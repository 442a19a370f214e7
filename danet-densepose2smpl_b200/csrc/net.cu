// Whole-network entry of the C ABI: loads a "network program" (the launch steps, buffer table and packed / folded
// weights that danet_b200.plan.Plan.export() writes for one batch size) and replays it -- the network half of
// DaNet.infer_net (models/danet/danet.py:78-98: img2iuv -> iuvmap_clean -> iuv2smpl up to `para`) for hosts without
// Python.  The Python plan runs each of its launches as one such step through danet_net_run_step, so both decode
// every launch with the same prepare / run_step and results are identical.  run_step is the one caller of the
// inference launchers (launchers.cuh), which check each step's arguments before they reach a kernel.
//
// Program layout (little endian, sections 16-byte aligned):
//   Header | u64 buf_bytes[n_buf] | {u64 off, u64 bytes} consts[n_const] | Out outs[n_out] | step stream | const payload
//   step = {u32 op, n_i, n_f, n_r} i32[n_i] f32[n_f] Ref[n_r];  Ref = {u32 kind (0 null, 1 buffer, 2 const, 3 input), u32 id, u64 off}
#include "launchers.cuh"
#include <string.h>

namespace danet {
namespace {

struct Header {
    char magic[8];                      // "DANETPRG"
    uint32_t version, batch, in_c, in_h, in_w, n_buf, n_const, n_out, n_step, precision, reserved0, reserved1;
    uint64_t steps_off, steps_bytes, payload_off, payload_bytes;
};
struct Ref { uint32_t kind, id; uint64_t off; };
struct OutRec { char name[32]; Ref ref; uint32_t elem_bytes; int32_t ndim; int32_t dims[4]; };
struct ConstRec { uint64_t off, bytes; };

enum { OP_INPUT = 1, OP_CONV_GROUP, OP_CONV_SIMT, OP_FUSE, OP_MAXPOOL, OP_AVGPOOL, OP_CLEAN_GLOBAL, OP_CLEAN_PARTS,
       OP_STN_PARAMS, OP_STN_SAMPLE, OP_LINEAR, OP_GCN_HEAD, OP_LAST };
constexpr int kDescInts = 11;           // danet_conv_desc fields, in declaration order

struct Step {
    uint32_t op = 0;
    std::vector<int32_t> i;
    std::vector<float> f;
    std::vector<void*> p;
    std::vector<danet_conv_problem> probs;     // OP_CONV_GROUP
    std::vector<danet_act> acts;               // OP_FUSE terms
    GcnArgs gcn;                               // OP_GCN_HEAD
};
struct Out { std::string name; void* ptr; uint64_t bytes; uint32_t elem_bytes; int32_t dims[4]; };

}  // namespace
}  // namespace danet

struct danet_net {
    int dev = 0;
    uint32_t batch = 0, in_c = 0, in_h = 0, in_w = 0, precision = 0;
    char* arena = nullptr;              // activations
    char* consts = nullptr;             // weights
    float* input = nullptr;             // static input [B,C,H,W] (the step list reads it; graph replay needs a fixed address)
    std::vector<danet::Step> steps;
    std::vector<danet::Out> outs;
    cudaGraphExec_t exec = nullptr;
    cudaStream_t own_stream = nullptr;  // danet_net_infer_host
    cudaStream_t blocking_stream = nullptr;   // graph replay for callers on the legacy default stream
    float* pinned = nullptr;
};

namespace danet {
namespace {

danet_conv_desc desc_of(const int32_t* v) {
    danet_conv_desc d;
    d.N = v[0]; d.H = v[1]; d.W = v[2]; d.Cin = v[3]; d.Cout = v[4]; d.ksize = v[5]; d.stride = v[6]; d.pad = v[7];
    d.wsets = v[8]; d.relu = v[9]; d.flags = v[10];
    return d;
}
danet_act act_of(void* const* p) {
    danet_act a;
    a.f32 = (float*)p[0]; a.hi = p[1]; a.lo = p[2];
    return a;
}

// number of (ints, refs) a step of kind `op` must carry; -1 = variable (checked in prepare)
int prepare(Step& s) {
    const size_t ni = s.i.size(), nr = s.p.size();
    const int32_t* I = s.i.data();
    void* const* P = s.p.data();
    switch (s.op) {
    case OP_INPUT: DANET_CHECK(ni == 4 && nr == 4, "net: malformed input step"); break;
    case OP_CONV_GROUP: {
        DANET_CHECK(ni >= 1 && I[0] >= 1 && I[0] <= 6 && ni == size_t(1 + kDescInts * I[0]) && nr == size_t(11 * I[0]),
                    "net: malformed conv group step");
        s.probs.resize(I[0]);
        for (int k = 0; k < I[0]; ++k) {
            danet_conv_problem& q = s.probs[k];
            q.d = desc_of(I + 1 + kDescInts * k);
            void* const* r = P + 11 * k;
            q.x = act_of(r); q.res = act_of(r + 3); q.y = act_of(r + 6);
            q.w_packed = r[9]; q.bias = (const float*)r[10];
        }
        break;
    }
    case OP_CONV_SIMT: DANET_CHECK(ni == size_t(kDescInts) && nr == 5, "net: malformed conv step"); break;
    case OP_FUSE: {
        DANET_CHECK(ni >= 6 && I[4] >= 1 && I[4] <= 4 && ni == size_t(6 + I[4]) && nr == size_t(3 * I[4] + 3),
                    "net: malformed fuse step");
        s.acts.resize(I[4]);
        for (int k = 0; k < I[4]; ++k) s.acts[k] = act_of(P + 3 * k);
        break;
    }
    case OP_MAXPOOL: DANET_CHECK(ni == 4 && nr == 6, "net: malformed maxpool step"); break;
    case OP_AVGPOOL: DANET_CHECK(ni == 3 && nr == 4, "net: malformed avgpool step"); break;
    case OP_CLEAN_GLOBAL: DANET_CHECK(ni == 8 && nr == 9, "net: malformed clean_global step"); break;
    case OP_CLEAN_PARTS: DANET_CHECK(ni == 4 && nr == 5, "net: malformed clean_parts step"); break;
    case OP_STN_PARAMS: DANET_CHECK(ni == 4 && s.f.size() == 1 && nr == 6, "net: malformed stn_params step"); break;
    case OP_STN_SAMPLE: DANET_CHECK(ni == 4 && nr == 7, "net: malformed stn_sample step"); break;
    case OP_LINEAR: DANET_CHECK(ni == 3 && nr == 5, "net: malformed linear step"); break;
    case OP_GCN_HEAD: {
        DANET_CHECK(ni == 11 && nr == 27, "net: malformed gcn_head step");
        GcnArgs& g = s.gcn;
        g.adj = (const float*)P[0];
        for (int l = 0; l < 5; ++l) {
            g.W[l] = (const float*)P[1 + l]; g.b[l] = (const float*)P[6 + l];
            g.bn_s[l] = (const float*)P[11 + l]; g.bn_t[l] = (const float*)P[16 + l];
            g.din[l] = I[1 + l]; g.dout[l] = I[6 + l];
        }
        g.head_w = (const float*)P[21]; g.head_b = (const float*)P[22]; g.mean_pose = (const float*)P[23];
        break;
    }
    default: DANET_CHECK(false, "net: unknown step kind %u", s.op);
    }
    return 0;
}

int run_step(const Step& s, cudaStream_t st) {
    const int32_t* I = s.i.data();
    void* const* P = s.p.data();
    switch (s.op) {
    case OP_INPUT: {
        danet_act y = act_of(P + 1);
        return nchw_to_nhwc(I[0], I[1], I[2], I[3], (const float*)P[0], &y, st);
    }
    case OP_CONV_GROUP: return danet_conv_tc_group(I[0], s.probs.data(), st);
    case OP_CONV_SIMT:
        return conv2d(desc_of(I), (const float*)P[0], (const float*)P[1], (const float*)P[2], (const float*)P[3],
                      (float*)P[4], st);
    case OP_FUSE: {
        danet_act y = act_of(P + 3 * I[4]);
        return fuse_sum(I[0], I[1], I[2], I[3], I[4], s.acts.data(), I + 6, I[5], &y, st);
    }
    case OP_MAXPOOL: {
        danet_act x = act_of(P), y = act_of(P + 3);
        return maxpool3x3s2(I[0], I[1], I[2], I[3], &x, &y, st);
    }
    case OP_AVGPOOL: {
        danet_act x = act_of(P);
        return danet_global_avgpool(I[0], I[1], I[2], &x, (float*)P[3], st);
    }
    case OP_CLEAN_GLOBAL: {
        danet_act body = act_of(P + 1);
        return iuv_clean_global(I[0], I[1], I[2], I[3], I[4], I[5], I[6], I[7], (const float*)P[0], &body,
                                (uint8_t*)P[4], (float*)P[5], (float*)P[6], (float*)P[7], (float*)P[8], st);
    }
    case OP_CLEAN_PARTS: {
        danet_act y = act_of(P + 1);
        return iuv_clean_parts(I[0], I[1], I[2], I[3], (const float*)P[0], &y, (float*)P[4], st);
    }
    case OP_STN_PARAMS:
        return stn_params(I[0], I[1], I[2], (const float*)P[0], (const uint8_t*)P[1], (const float*)P[2],
                          (const float*)P[3], s.f[0], I[3], (float*)P[4], (float*)P[5], st);
    case OP_STN_SAMPLE: {
        danet_act xd = act_of(P), crops = act_of(P + 4);
        return stn_sample(I[0], I[1], I[2], &xd, (const float*)P[3], I[3], &crops, st);
    }
    case OP_LINEAR:
        return danet_linear(I[0], I[1], I[2], (const float*)P[0], (const float*)P[1], (const float*)P[2],
                            (const float*)P[3], (float*)P[4], st);
    case OP_GCN_HEAD:
        return gcn_pose_head(I[0], s.gcn, (const float*)P[24], (const float*)P[25], (float*)P[26], st);
    }
    set_error("net: unknown step kind %u", s.op);
    return -1;
}

int run_steps(const danet_net* net, cudaStream_t st) {
    for (size_t k = 0; k < net->steps.size(); ++k) {
        int rc = run_step(net->steps[k], st);
        if (rc != 0) return rc;                 // the failing entry has set the message
    }
    return 0;
}

struct DeviceGuard {                            // kernels, buffers and stream must belong to the program's device
    int prev = -1; bool ok = true;
    explicit DeviceGuard(int dev) { ok = cudaGetDevice(&prev) == cudaSuccess && (prev == dev || cudaSetDevice(dev) == cudaSuccess); if (prev == dev) prev = -1; }
    ~DeviceGuard() { if (prev >= 0) cudaSetDevice(prev); }
};

void free_net(danet_net* n) {
    if (!n) return;
    if (n->exec) cudaGraphExecDestroy(n->exec);
    if (n->own_stream) cudaStreamDestroy(n->own_stream);
    if (n->blocking_stream) cudaStreamDestroy(n->blocking_stream);
    if (n->pinned) cudaFreeHost(n->pinned);
    cudaFree(n->arena); cudaFree(n->consts); cudaFree(n->input);
    delete n;
}

}  // namespace
}  // namespace danet

using namespace danet;

extern "C" int danet_net_load(const void* program, uint64_t bytes, danet_net_t* out) {
    DANET_CHECK(program && out, "net_load: null argument");
    const char* base = (const char*)program;
    DANET_CHECK(bytes >= sizeof(Header), "net_load: truncated program");
    Header h;
    memcpy(&h, base, sizeof(h));
    DANET_CHECK(memcmp(h.magic, "DANETPRG", 8) == 0, "net_load: not a network program (bad magic)");
    DANET_CHECK(h.version == 1, "net_load: program version %u, this library reads version 1", h.version);
    uint64_t off = sizeof(Header);
    const uint64_t tables = uint64_t(h.n_buf) * 8 + uint64_t(h.n_const) * sizeof(ConstRec) + uint64_t(h.n_out) * sizeof(OutRec);
    DANET_CHECK(off + tables <= bytes && h.steps_off + h.steps_bytes <= bytes && h.payload_off + h.payload_bytes <= bytes,
                "net_load: truncated program");
    std::vector<uint64_t> buf_bytes(h.n_buf);
    memcpy(buf_bytes.data(), base + off, h.n_buf * 8ull); off += h.n_buf * 8ull;
    std::vector<ConstRec> crec(h.n_const);
    memcpy(crec.data(), base + off, h.n_const * sizeof(ConstRec)); off += h.n_const * sizeof(ConstRec);
    std::vector<OutRec> orec(h.n_out);
    memcpy(orec.data(), base + off, h.n_out * sizeof(OutRec));

    int cur_dev = 0;
    DANET_CUDA(cudaGetDevice(&cur_dev));
    danet_net* net = new danet_net();
    net->dev = cur_dev;
    net->batch = h.batch; net->in_c = h.in_c; net->in_h = h.in_h; net->in_w = h.in_w; net->precision = h.precision;
    // one arena for the activations, one for the constants (256-byte aligned members: TMA bases need 16)
    std::vector<uint64_t> boff(h.n_buf), coff(h.n_const);
    uint64_t total = 0;
    for (uint32_t k = 0; k < h.n_buf; ++k) { boff[k] = total; total += align_up((int64_t)buf_bytes[k], 256); }
    uint64_t ctotal = 0;
    for (uint32_t k = 0; k < h.n_const; ++k) {
        if (crec[k].off + crec[k].bytes > bytes) { free_net(net); DANET_CHECK(false, "net_load: constant %u out of range", k); }
        coff[k] = ctotal; ctotal += align_up((int64_t)crec[k].bytes, 256);
    }
    cudaError_t e = cudaMalloc((void**)&net->arena, total + 256);
    if (e == cudaSuccess) e = cudaMemset(net->arena, 0, total + 256);
    if (e == cudaSuccess) e = cudaMalloc((void**)&net->consts, ctotal + 256);
    if (e == cudaSuccess) e = cudaMalloc((void**)&net->input, sizeof(float) * size_t(h.batch) * h.in_c * h.in_h * h.in_w + 256);
    for (uint32_t k = 0; k < h.n_const && e == cudaSuccess; ++k)
        e = cudaMemcpy(net->consts + coff[k], base + crec[k].off, crec[k].bytes, cudaMemcpyHostToDevice);
    if (e != cudaSuccess) { free_net(net); DANET_CHECK(false, "net_load: device memory: %s", cudaGetErrorString(e)); }

    bool bad = false;
    auto resolve = [&](const Ref& r, uint64_t need) -> void* {
        switch (r.kind) {
        case 0: return nullptr;
        case 1: if (r.id >= h.n_buf || r.off + need > buf_bytes[r.id]) { bad = true; return nullptr; } return net->arena + boff[r.id] + r.off;
        case 2: if (r.id >= h.n_const || r.off + need > crec[r.id].bytes) { bad = true; return nullptr; } return net->consts + coff[r.id] + r.off;
        case 3: return net->input;
        }
        bad = true;
        return nullptr;
    };
    for (uint32_t k = 0; k < h.n_out; ++k) {
        Out o;
        char nm[33]; memcpy(nm, orec[k].name, 32); nm[32] = 0;
        o.name = nm; o.elem_bytes = orec[k].elem_bytes;
        uint64_t n = 1;
        for (int d = 0; d < 4; ++d) { o.dims[d] = d < orec[k].ndim ? orec[k].dims[d] : 1; n *= (uint64_t)o.dims[d]; }
        o.bytes = n * o.elem_bytes;
        o.ptr = resolve(orec[k].ref, o.bytes);
        net->outs.push_back(o);
    }
    // step stream
    const char* sp = base + h.steps_off;
    const char* se = sp + h.steps_bytes;
    net->steps.resize(h.n_step);
    int rc = 0;
    for (uint32_t k = 0; k < h.n_step && rc == 0 && !bad; ++k) {
        uint32_t hd[4];
        if (sp + 16 > se) { bad = true; break; }
        memcpy(hd, sp, 16); sp += 16;
        const uint64_t need = 4ull * hd[1] + 4ull * hd[2] + sizeof(Ref) * uint64_t(hd[3]);
        if (uint64_t(se - sp) < need) { bad = true; break; }
        Step& s = net->steps[k];
        s.op = hd[0];
        s.i.resize(hd[1]); memcpy(s.i.data(), sp, 4ull * hd[1]); sp += 4ull * hd[1];
        s.f.resize(hd[2]); memcpy(s.f.data(), sp, 4ull * hd[2]); sp += 4ull * hd[2];
        s.p.resize(hd[3]);
        for (uint32_t r = 0; r < hd[3]; ++r) { Ref ref; memcpy(&ref, sp, sizeof(Ref)); sp += sizeof(Ref); s.p[r] = resolve(ref, 0); }
        rc = prepare(s);
    }
    if (bad || rc != 0) {
        free_net(net);
        if (bad) set_error("net_load: malformed program (reference or step out of range)");
        return -1;
    }
    *out = net;
    return 0;
}

extern "C" int danet_net_load_file(const char* path, danet_net_t* out) {
    DANET_CHECK(path && out, "net_load_file: null argument");
    FILE* f = fopen(path, "rb");
    DANET_CHECK(f != nullptr, "net_load_file: cannot open %s", path);
    fseek(f, 0, SEEK_END);
    long n = ftell(f);
    fseek(f, 0, SEEK_SET);
    std::vector<char> blob(n > 0 ? (size_t)n : 0);
    size_t got = n > 0 ? fread(blob.data(), 1, (size_t)n, f) : 0;
    fclose(f);
    DANET_CHECK(n > 0 && got == (size_t)n, "net_load_file: short read of %s", path);
    return danet_net_load(blob.data(), (uint64_t)n, out);
}

extern "C" int danet_net_destroy(danet_net_t net) {
    if (net) { DeviceGuard g(net->dev); free_net(net); }
    return 0;
}

extern "C" int danet_net_info(danet_net_t net, int32_t* batch, int32_t* chw, int32_t* n_outputs, int32_t* n_steps) {
    DANET_CHECK(net, "net_info: null handle");
    if (batch) *batch = (int32_t)net->batch;
    if (chw) { chw[0] = (int32_t)net->in_c; chw[1] = (int32_t)net->in_h; chw[2] = (int32_t)net->in_w; }
    if (n_outputs) *n_outputs = (int32_t)net->outs.size();
    if (n_steps) *n_steps = (int32_t)net->steps.size();
    return 0;
}

extern "C" const char* danet_net_output_name(danet_net_t net, int32_t index) {
    if (!net || index < 0 || (size_t)index >= net->outs.size()) return nullptr;
    return net->outs[index].name.c_str();
}

extern "C" int danet_net_output(danet_net_t net, const char* name, void** dev_ptr, uint64_t* bytes, int32_t* dims,
                                int32_t* elem_bytes) {
    DANET_CHECK(net && name, "net_output: null argument");
    for (const Out& o : net->outs) {
        if (o.name == name) {
            if (dev_ptr) *dev_ptr = o.ptr;
            if (bytes) *bytes = o.bytes;
            if (dims) for (int d = 0; d < 4; ++d) dims[d] = o.dims[d];
            if (elem_bytes) *elem_bytes = (int32_t)o.elem_bytes;
            return 0;
        }
    }
    DANET_CHECK(false, "net_output: the program has no output named '%s'", name);
}

extern "C" int danet_net_infer(danet_net_t net, const float* images, int32_t flags, danet_stream_t stream) {
    DANET_CHECK(net && images, "net_infer: null argument");
    DeviceGuard g(net->dev);
    DANET_CHECK(g.ok, "net_infer: cannot select device %d", net->dev);
    cudaStream_t st = (cudaStream_t)stream;
    if (st == nullptr && (flags & DANET_NET_GRAPH)) {
        // the legacy default stream cannot be captured: a BLOCKING stream of our own keeps its ordering
        // (implicit synchronisation with the legacy stream, both ways)
        if (!net->blocking_stream) DANET_CUDA(cudaStreamCreate(&net->blocking_stream));
        st = net->blocking_stream;
    }
    const size_t in_bytes = sizeof(float) * size_t(net->batch) * net->in_c * net->in_h * net->in_w;
    DANET_CUDA(cudaMemcpyAsync(net->input, images, in_bytes, cudaMemcpyDefault, st));
    if (!(flags & DANET_NET_GRAPH)) return run_steps(net, st);
    if (!net->exec) {
        int rc = run_steps(net, st);            // first-use work (function attributes, scheduler counters) outside the capture
        if (rc != 0) return rc;
        cudaGraph_t graph = nullptr;
        DANET_CUDA(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
        rc = run_steps(net, st);
        cudaError_t e = cudaStreamEndCapture(st, &graph);
        if (rc != 0) { if (graph) cudaGraphDestroy(graph); return rc; }
        DANET_CHECK(e == cudaSuccess && graph, "net_infer: stream capture failed: %s", cudaGetErrorString(e));
        e = cudaGraphInstantiate(&net->exec, graph, 0);
        cudaGraphDestroy(graph);
        DANET_CHECK(e == cudaSuccess, "net_infer: cudaGraphInstantiate: %s", cudaGetErrorString(e));
    }
    DANET_CUDA(cudaGraphLaunch(net->exec, st));
    return 0;
}

extern "C" int danet_net_infer_host(danet_net_t net, const float* images_host, int32_t flags) {
    DANET_CHECK(net && images_host, "net_infer_host: null argument");
    DeviceGuard g(net->dev);
    DANET_CHECK(g.ok, "net_infer_host: cannot select device %d", net->dev);
    const size_t in_bytes = sizeof(float) * size_t(net->batch) * net->in_c * net->in_h * net->in_w;
    if (!net->own_stream) DANET_CUDA(cudaStreamCreateWithFlags(&net->own_stream, cudaStreamNonBlocking));
    if (!net->pinned) DANET_CUDA(cudaMallocHost((void**)&net->pinned, in_bytes));
    memcpy(net->pinned, images_host, in_bytes);
    int rc = danet_net_infer(net, net->pinned, flags, (danet_stream_t)net->own_stream);
    if (rc != 0) return rc;
    DANET_CUDA(cudaStreamSynchronize(net->own_stream));
    return 0;
}

extern "C" int danet_net_run_step(uint32_t op, int32_t n_i, const int32_t* i, int32_t n_f, const float* f, int32_t n_p,
                                  void* const* p, danet_stream_t stream) {
    DANET_CHECK(n_i >= 0 && n_f >= 0 && n_p >= 0 && (i || !n_i) && (f || !n_f) && (p || !n_p), "net_run_step: null argument");
    Step s;
    s.op = op;
    s.i.assign(i, i + n_i);
    s.f.assign(f, f + n_f);
    s.p.assign(p, p + n_p);
    int rc = prepare(s);
    return rc != 0 ? rc : run_step(s, (cudaStream_t)stream);
}

extern "C" int danet_net_read_output(danet_net_t net, const char* name, void* host_dst, uint64_t bytes) {
    DANET_CHECK(net && host_dst, "net_read_output: null argument");
    void* p = nullptr; uint64_t n = 0;
    int rc = danet_net_output(net, name, &p, &n, nullptr, nullptr);
    if (rc != 0) return rc;
    DANET_CHECK(bytes == n, "net_read_output: '%s' holds %llu bytes, caller asked for %llu", name, (unsigned long long)n,
                (unsigned long long)bytes);
    DeviceGuard g(net->dev);
    if (net->own_stream) DANET_CUDA(cudaStreamSynchronize(net->own_stream));
    DANET_CUDA(cudaMemcpy(host_dst, p, n, cudaMemcpyDeviceToHost));
    return 0;
}
