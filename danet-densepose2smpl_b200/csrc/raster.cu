// IUV rasteriser for sm_90a.  Replaces utils/renderer.py:207-298 (IUV_Renderer.verts2uvimg /
// camera_matrix) and the third-party neural_renderer forward pass behind it (projection,
// vertices_to_faces, forward_face_index_map kernels, texture sampling, vertical flip), and
// optionally fuses utils/iuvmap.py:103-151 (iuv_img2map) into the resolve pass.
//
// The upstream kernel loops every pixel over all 13774 faces (43 M tests / image).  Here:
//   k_project   thread per (image, mesh vertex): gather SMPL vertex, project to NDC
//   k_faces     thread per (image, face): back-face cull, bounding box (+1 px guard band), the
//               same edge tests / barycentric inverse / perspective depth as upstream for the
//               pixels inside the box, then a 64-bit atomicMin of (depth bits << 32 | face id)
//               on a per-pixel key -- strict z-min with lowest-face-id tie break, i.e. exactly
//               the winner the sequential upstream loop keeps
//   k_resolve   thread per output pixel: decode winner, emit texture, vertical flip, optional
//               25/25/25/15-channel maps
// All geometry uses __f*_rn intrinsics (no FMA contraction) in the order oracle/raster.c uses,
// so the integer winner (face id -> part id) is bit-exact against the CPU restatement.
// danet_raster_iuv_select renders a per-image subset (danet.py:163-165): k_project and k_faces skip the other images,
// whose z-buffer stays cleared, so k_resolve writes them as the zero image and its maps.
#include "common.cuh"

struct danet_raster {
    int nv, nmv, nf, orig, S, tex_mode;
    float focal, near_, far_;
    int* vmap; int* faces; float* tex;
};

namespace danet {

__device__ __forceinline__ float fm(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float fa(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float fs(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ float fd(float a, float b) { return __fdiv_rn(a, b); }

__global__ void k_project(int B, int nv, int nmv, const float* __restrict__ verts,
                          const float* __restrict__ cam, const int* __restrict__ vmap, float focal,
                          int orig, const uint8_t* __restrict__ select, float* __restrict__ pv) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B * nmv) return;
    const int b = i / nmv, k = i % nmv;
    if (select && !select[b]) return;                 // unselected image: k_faces never reads its vertices
    const float* v = verts + ((size_t)b * nv + vmap[k]) * 3;
    const float* c = cam + (size_t)b * 3;
    const float o = (float)orig;
    const float tz = fd(fm(2.0f, focal), fa(fm(o, c[0]), 1e-9f));
    const float x = fa(v[0], c[1]);
    const float y = fa(v[1], c[2]);
    const float z = fa(v[2], tz);
    const float zz = fa(z, 1e-9f);
    const float x_ = fd(x, zz), y_ = fd(y, zz);
    const float ctr = fd(o, 2.0f);
    float u = fa(fm(x_, focal), ctr);
    float w = fa(fm(y_, focal), ctr);
    w = fs(o, w);
    u = fd(fm(2.0f, fs(u, ctr)), o);
    w = fd(fm(2.0f, fs(w, ctr)), o);
    pv[(size_t)i * 3 + 0] = u;
    pv[(size_t)i * 3 + 1] = w;
    pv[(size_t)i * 3 + 2] = z;
}

__global__ void k_faces(int B, int nmv, int nf, int S, float near_, float far_,
                        const float* __restrict__ pv, const int* __restrict__ faces,
                        const uint8_t* __restrict__ select, unsigned long long* __restrict__ zbuf) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B * nf) return;
    const int b = i / nf, f = i % nf;
    if (select && !select[b]) return;                 // its z-buffer stays cleared: k_resolve writes background
    float face[9];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const float* p = pv + ((size_t)b * nmv + faces[f * 3 + k]) * 3;
        face[3 * k] = p[0]; face[3 * k + 1] = p[1]; face[3 * k + 2] = p[2];
    }
    // non-finite coordinates can never win upstream's z-test either (NaN compares false)
#pragma unroll
    for (int k = 0; k < 9; ++k) if (!isfinite(face[k])) return;
    // back-face cull (fill_back=False)
    if (fm(fs(face[7], face[1]), fs(face[3], face[0])) < fm(fs(face[4], face[1]), fs(face[6], face[0]))) return;
    const float is = (float)S;
    float p[3][2];
#pragma unroll
    for (int n = 0; n < 3; ++n)
#pragma unroll
        for (int d = 0; d < 2; ++d) p[n][d] = fm(0.5f, fs(fa(fm(face[3 * n + d], is), is), 1.0f));
    float fi[9] = {
        fs(p[1][1], p[2][1]), fs(p[2][0], p[1][0]), fs(fm(p[1][0], p[2][1]), fm(p[2][0], p[1][1])),
        fs(p[2][1], p[0][1]), fs(p[0][0], p[2][0]), fs(fm(p[2][0], p[0][1]), fm(p[0][0], p[2][1])),
        fs(p[0][1], p[1][1]), fs(p[1][0], p[0][0]), fs(fm(p[0][0], p[1][1]), fm(p[1][0], p[0][1]))};
    const float den = fa(fa(fm(p[2][0], fs(p[0][1], p[1][1])), fm(p[0][0], fs(p[1][1], p[2][1]))),
                         fm(p[1][0], fs(p[2][1], p[0][1])));
#pragma unroll
    for (int k = 0; k < 9; ++k) fi[k] = fd(fi[k], den);
    // pixel-space bounding box with a 1-pixel guard band (edge tests are evaluated in fp32)
    const float pxmin = fminf(p[0][0], fminf(p[1][0], p[2][0])), pxmax = fmaxf(p[0][0], fmaxf(p[1][0], p[2][0]));
    const float pymin = fminf(p[0][1], fminf(p[1][1], p[2][1])), pymax = fmaxf(p[0][1], fmaxf(p[1][1], p[2][1]));
    if (pxmax < -1.0f || pymax < -1.0f || pxmin > is || pymin > is) return;
    const int x0 = max(0, (int)floorf(pxmin) - 1), x1 = min(S - 1, (int)ceilf(pxmax) + 1);
    const int y0 = max(0, (int)floorf(pymin) - 1), y1 = min(S - 1, (int)ceilf(pymax) + 1);
    unsigned long long* zb = zbuf + (size_t)b * S * S;
    for (int yi = y0; yi <= y1; ++yi) {
        const float yp = fd((float)(2 * yi + 1 - S), is);
        for (int xi = x0; xi <= x1; ++xi) {
            const float xp = fd((float)(2 * xi + 1 - S), is);
            if ((fm(fs(yp, face[1]), fs(face[3], face[0])) < fm(fs(xp, face[0]), fs(face[4], face[1]))) ||
                (fm(fs(yp, face[4]), fs(face[6], face[3])) < fm(fs(xp, face[3]), fs(face[7], face[4]))) ||
                (fm(fs(yp, face[7]), fs(face[0], face[6])) < fm(fs(xp, face[6]), fs(face[1], face[7]))))
                continue;
            float w[3], wsum = 0.0f;
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                float wk = fa(fa(fm(fi[3 * k], (float)xi), fm(fi[3 * k + 1], (float)yi)), fi[3 * k + 2]);
                wk = wk > 0.0f ? wk : 0.0f;
                wk = wk < 1.0f ? wk : 1.0f;
                w[k] = wk;
                wsum = fa(wsum, wk);
            }
#pragma unroll
            for (int k = 0; k < 3; ++k) w[k] = fd(w[k], wsum);
            const float zp = fd(1.0f, fa(fa(fd(w[0], face[2]), fd(w[1], face[5])), fd(w[2], face[8])));
            if (zp <= near_ || far_ <= zp) continue;
            if (!(zp < far_)) continue;                       // NaN guard (never selected upstream)
            const unsigned long long key = ((unsigned long long)__float_as_uint(zp) << 32) | (unsigned)f;
            atomicMin(zb + yi * S + xi, key);
        }
    }
}

__device__ __forceinline__ void emit_maps(float I, float U, float V, int b, int pix, int HW,
                                          float* mu, float* mv, float* mi, float* ma) {
    // utils/iuvmap.py:103-151: part = round(I*24); one-hot over 25; U,V masked; 15-class ann merge
    const float part = rintf(I * 24.0f);
    const int ann_of[25] = {0, 1, 1, 2, 3, 4, 5, 6, 7, 6, 7, 8, 9, 8, 9, 10, 11, 10, 11, 12, 13, 12, 13, 14, 14};
    for (int c = 0; c < 25; ++c) {
        const float oh = (part == (float)c) ? 1.0f : 0.0f;
        const size_t o = ((size_t)b * 25 + c) * HW + pix;
        if (mi) mi[o] = oh;
        if (mu) mu[o] = oh * U;
        if (mv) mv[o] = oh * V;
    }
    if (ma) {
        for (int a = 0; a < 15; ++a) ma[((size_t)b * 15 + a) * HW + pix] = 0.0f;
        if (part >= 0.0f && part <= 24.0f) ma[((size_t)b * 15 + ann_of[(int)part]) * HW + pix] = 1.0f;
    }
}

__global__ void k_resolve(int B, int S, int nf, int tex_mode, const unsigned long long* __restrict__ zbuf,
                          const float* __restrict__ tex, float* __restrict__ img, int* __restrict__ face_idx,
                          float* mu, float* mv, float* mi, float* ma) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B * S * S) return;
    const int b = i / (S * S), pix = i % (S * S), yo = pix / S, xi = pix % S;
    const int yi = S - 1 - yo;                                  // vertical flip
    const unsigned long long key = zbuf[(size_t)b * S * S + yi * S + xi];
    const int f = (key == ~0ull) ? -1 : (int)(key & 0xffffffffu);
    float c[3] = {0.f, 0.f, 0.f};
    if (f >= 0) {
        if (tex_mode == 0) {
            c[0] = tex[(size_t)f * 3]; c[1] = tex[(size_t)f * 3 + 1]; c[2] = tex[(size_t)f * 3 + 2];
        } else {
            const float fr = fs(-1e-3f, (float)(int)(-1e-3f));
            for (int ch = 0; ch < 3; ++ch) {
                float val = 0.0f;
                for (int pn = 0; pn < 8; ++pn) {
                    float ww = 1.0f; int isc = 0;
                    for (int k = 0; k < 3; ++k) {
                        if (((pn >> k) % 2) == 0) ww = fm(ww, fs(1.0f, fr));
                        else { ww = fm(ww, fr); isc += 1; }
                    }
                    int ff = f + isc; if (ff > nf - 1) ff = nf - 1;
                    val = fa(val, fm(ww, tex[(size_t)ff * 3 + ch]));
                }
                c[ch] = val;
            }
        }
    }
    const int HW = S * S;
    if (img) {
        img[((size_t)b * 3 + 0) * HW + pix] = c[0];
        img[((size_t)b * 3 + 1) * HW + pix] = c[1];
        img[((size_t)b * 3 + 2) * HW + pix] = c[2];
    }
    if (face_idx) face_idx[(size_t)b * HW + pix] = f;
    if (mu || mv || mi || ma) emit_maps(c[0], c[1], c[2], b, pix, HW, mu, mv, mi, ma);
}

__global__ void k_img2map(int B, int HW, const float* __restrict__ img, float* mu, float* mv, float* mi, float* ma) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B * HW) return;
    const int b = i / HW, pix = i % HW;
    emit_maps(img[((size_t)b * 3) * HW + pix], img[((size_t)b * 3 + 1) * HW + pix],
              img[((size_t)b * 3 + 2) * HW + pix], b, pix, HW, mu, mv, mi, ma);
}

// the rasteriser's workspace: projected mesh vertices, then the z-buffer keys; a null base only sizes it
struct RasterWs {
    float* pv; unsigned long long* zbuf; int64_t bytes;
    RasterWs(const danet_raster* h, int B, void* base) {
        WsCarve c{(char*)base};
        pv = c.take<float>((int64_t)B * h->nmv * 3);
        zbuf = c.take<unsigned long long>((int64_t)B * h->S * h->S);
        bytes = c.bytes;
    }
};

}  // namespace danet

using namespace danet;

extern "C" int danet_raster_create(const danet_raster_desc* d, danet_raster_t* out) {
    DANET_CHECK(d && out, "danet_raster_create: null argument");
    DANET_CHECK(d->vert_mapping && d->faces && d->textures, "danet_raster_create: missing mesh array");
    DANET_CHECK(d->out_size > 0 && d->out_size <= 1024 && d->orig_size > 0, "danet_raster_create: bad sizes");
    for (int i = 0; i < d->num_mesh_verts; ++i)
        DANET_CHECK(d->vert_mapping[i] >= 0 && d->vert_mapping[i] < d->num_smpl_verts,
                    "danet_raster_create: vert_mapping[%d]=%d out of range", i, d->vert_mapping[i]);
    for (int i = 0; i < d->num_faces * 3; ++i)
        DANET_CHECK(d->faces[i] >= 0 && d->faces[i] < d->num_mesh_verts,
                    "danet_raster_create: face index %d out of range", d->faces[i]);
    auto* h = new danet_raster();
    h->nv = d->num_smpl_verts; h->nmv = d->num_mesh_verts; h->nf = d->num_faces;
    h->orig = d->orig_size; h->S = d->out_size; h->tex_mode = d->tex_mode;
    h->focal = d->focal_length; h->near_ = d->near_plane; h->far_ = d->far_plane;
    h->vmap = nullptr; h->faces = nullptr; h->tex = nullptr;
    int rc = upload(&h->vmap, d->vert_mapping, (size_t)h->nmv);
    rc |= upload(&h->faces, d->faces, (size_t)h->nf * 3);
    rc |= upload(&h->tex, d->textures, (size_t)h->nf * 3);
    if (rc != 0) { danet_raster_destroy(h); return -2; }
    *out = h;
    return 0;
}

extern "C" int danet_raster_destroy(danet_raster_t h) {
    if (!h) return 0;
    cudaFree(h->vmap); cudaFree(h->faces); cudaFree(h->tex);
    delete h;
    return 0;
}

extern "C" int64_t danet_raster_workspace_bytes(danet_raster_t h, int32_t B) {
    if (!h || B <= 0) return 0;
    return RasterWs(h, B, nullptr).bytes;
}

extern "C" int danet_raster_iuv_select(danet_raster_t h, int32_t B, const float* verts, const float* cam,
                                       const uint8_t* select, float* img, int32_t* face_idx, float* maps_u, float* maps_v,
                                       float* maps_i, float* maps_ann, void* workspace, danet_stream_t stream_) {
    DANET_CHECK(h, "danet_raster_iuv: null handle");
    DANET_CHECK(B > 0, "danet_raster_iuv: empty batch (B=%d)", B);
    DANET_CHECK(verts && cam && workspace, "danet_raster_iuv: null input/workspace pointer");
    cudaStream_t stream = (cudaStream_t)stream_;
    const RasterWs ws(h, B, workspace);
    DANET_CUDA(cudaMemsetAsync(ws.zbuf, 0xff, (size_t)B * h->S * h->S * 8, stream));
    k_project<<<cdiv(B * h->nmv, 256), 256, 0, stream>>>(B, h->nv, h->nmv, verts, cam, h->vmap, h->focal, h->orig, select, ws.pv);
    DANET_LAUNCH_CHECK();
    k_faces<<<cdiv(B * h->nf, 128), 128, 0, stream>>>(B, h->nmv, h->nf, h->S, h->near_, h->far_, ws.pv, h->faces, select, ws.zbuf);
    DANET_LAUNCH_CHECK();
    k_resolve<<<cdiv(B * h->S * h->S, 256), 256, 0, stream>>>(B, h->S, h->nf, h->tex_mode, ws.zbuf, h->tex, img, face_idx,
                                                            maps_u, maps_v, maps_i, maps_ann);
    DANET_LAUNCH_CHECK();
    return 0;
}

extern "C" int danet_raster_iuv(danet_raster_t h, int32_t B, const float* verts, const float* cam, float* img,
                                int32_t* face_idx, float* maps_u, float* maps_v, float* maps_i, float* maps_ann,
                                void* workspace, danet_stream_t stream) {
    return danet_raster_iuv_select(h, B, verts, cam, nullptr, img, face_idx, maps_u, maps_v, maps_i, maps_ann, workspace,
                                   stream);
}

extern "C" int danet_iuv_img2map(int32_t B, int32_t S, const float* img, float* maps_u, float* maps_v,
                                 float* maps_i, float* maps_ann, danet_stream_t stream) {
    DANET_CHECK(B >= 0 && S > 0, "danet_iuv_img2map: bad sizes");
    if (B == 0) return 0;
    DANET_CHECK(img, "danet_iuv_img2map: null image");
    k_img2map<<<cdiv(B * S * S, 256), 256, 0, (cudaStream_t)stream>>>(B, S * S, img, maps_u, maps_v, maps_i, maps_ann);
    DANET_LAUNCH_CHECK();
    return 0;
}
