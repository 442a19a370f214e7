"""IUV renderer with the reference's call surface (utils/renderer.py:202-298 IUV_Renderer),
executed by csrc/raster.cu through the C ABI (projection + binned z-min rasterisation + resolve,
optionally emitting the 25/25/25/15-channel maps of utils/iuvmap.py:103-151 in the same pass)."""
import ctypes
import os

import numpy as np
import torch

from . import _lib


def load_dp_mesh(path="./data/UV_data/UV_Processed.mat"):
    """What DensePoseMethods.__init__ reads (utils/densepose_methods.py:16-29)."""
    if not os.path.exists(path):
        raise ValueError("%s does not exist (DensePose UV data, reference README.md:60-65)" % path)
    import scipy.io as sio
    m = sio.loadmat(path)
    return {"All_vertices": m["All_vertices"][0], "FacesDensePose": m["All_Faces"] - 1,
            "FaceIndices": np.array(m["All_FaceIndices"]).squeeze(),
            "U_norm": m["All_U_norm"].squeeze(), "V_norm": m["All_V_norm"].squeeze()}


class IUV_Renderer(object):
    """Renderer for generating IUV maps (same attributes as the reference object)."""

    def __init__(self, orig_size=224, out_size=56, focal_length=5000., mesh=None, tex_mode=0,
                 num_smpl_verts=6890):
        self.orig_size = orig_size
        self.out_size = out_size
        self.focal_length = focal_length
        self.tex_mode = tex_mode
        K = np.array([[self.focal_length, 0., self.orig_size / 2.],
                      [0., self.focal_length, self.orig_size / 2.],
                      [0., 0., 1.]])
        if self.orig_size != 224:                           # renderer.py:222-227
            s = self.orig_size / float(224)
            K[0, 0] *= s; K[1, 1] *= s; K[0, 2] *= s; K[1, 2] *= s
        self._focal_eff = float(K[0, 0])
        self.K = torch.FloatTensor(K[None, :, :])
        self.R = torch.FloatTensor(np.eye(3)[None, :, :])
        self.t = torch.FloatTensor(np.array([0, 0, 5])[None, None, :])
        self.coco_plus2coco = [14, 15, 16, 17, 18, 9, 8, 10, 7, 11, 6, 3, 2, 4, 1, 5, 0]
        DP = load_dp_mesh() if mesh is None else mesh
        vert_mapping = np.asarray(DP["All_vertices"]).astype("int64") - 1
        self.vert_mapping = torch.from_numpy(vert_mapping)
        faces = np.asarray(DP["FacesDensePose"])
        self.faces = torch.from_numpy(faces[None].astype(np.int32))
        num_part = float(np.max(DP["FaceIndices"]))
        U, V = np.asarray(DP["U_norm"]), np.asarray(DP["V_norm"])
        textures = np.stack([np.asarray(DP["FaceIndices"]) / num_part, U[faces].mean(1), V[faces].mean(1)], -1)
        self.textures = torch.from_numpy(textures[None, :, None, None, None, :].astype(np.float32))
        self.num_smpl_verts = num_smpl_verts
        self._handles = {}
        self._ws = {}

    def _handle(self, device):
        key = device.index if device.index is not None else torch.cuda.current_device()
        if key in self._handles:
            return self._handles[key]
        vm = np.ascontiguousarray(self.vert_mapping.numpy(), dtype=np.int32)
        fc = np.ascontiguousarray(self.faces[0].numpy(), dtype=np.int32)
        tx = np.ascontiguousarray(self.textures.reshape(-1, 3).numpy(), dtype=np.float32)
        d = _lib.RasterDesc()
        d.num_smpl_verts = self.num_smpl_verts
        d.num_mesh_verts = vm.shape[0]
        d.vert_mapping = vm.ctypes.data_as(ctypes.c_void_p)
        d.num_faces = fc.shape[0]
        d.faces = fc.ctypes.data_as(ctypes.c_void_p)
        d.textures = tx.ctypes.data_as(ctypes.c_void_p)
        d.orig_size = self.orig_size
        d.out_size = self.out_size
        d.focal_length = self._focal_eff
        d.near_plane, d.far_plane = 0.1, 100.0
        d.tex_mode = self.tex_mode
        h = ctypes.c_void_p()
        with torch.cuda.device(key):
            _lib.check(_lib.load().danet_raster_create(ctypes.byref(d), ctypes.byref(h)), "raster_create")
        self._handles[key] = h
        return h

    def __del__(self):
        try:
            for h in self._handles.values():
                _lib.load().danet_raster_destroy(h)
        except Exception:
            pass

    @torch.no_grad()
    def _render(self, verts, cam, want_maps=False, want_face_idx=False, select=None):
        """select: optional uint8 [B] on the device; images with select == 0 are not rasterised and come out as
        background (the zero image and its maps), as danet.py:163-165 renders only the has_iuv images."""
        _lib.require_cuda(verts, "verts")
        dev = verts.device
        B = verts.size(0)
        if verts.shape[1] != self.num_smpl_verts:
            raise ValueError("verts2uvimg: expected [B,%d,3] vertices" % self.num_smpl_verts)
        verts_c = verts.detach().float().contiguous()
        cam_c = cam.detach().to(dev).float().contiguous()
        S = self.out_size
        if B == 0:                                       # empty batch: empty outputs, nothing to launch
            return (torch.empty(0, 3, S, S, device=dev), torch.empty(0, S, S, dtype=torch.int32, device=dev) if want_face_idx else None,
                    [torch.empty(0, c, S, S, device=dev) for c in (25, 25, 25, 15)] if want_maps else [None] * 4)
        with torch.cuda.device(dev):
            h = self._handle(dev)
            need = int(_lib.load().danet_raster_workspace_bytes(h, B))
            ws = self._ws.get(dev.index)
            if ws is None or ws.numel() < need:
                ws = _lib.workspace(need, dev)
                self._ws[dev.index] = ws
            img = torch.empty(B, 3, S, S, device=dev)
            fidx = torch.empty(B, S, S, dtype=torch.int32, device=dev) if want_face_idx else None
            maps = [torch.empty(B, c, S, S, device=dev) for c in (25, 25, 25, 15)] if want_maps else [None] * 4
            if select is None:
                _lib.call("raster_iuv", h, B, _lib.ptr(verts_c), _lib.ptr(cam_c), _lib.ptr(img), _lib.ptr(fidx),
                          *map(_lib.ptr, maps), _lib.ptr(ws))
            else:
                _lib.call("raster_iuv_select", h, B, _lib.ptr(verts_c), _lib.ptr(cam_c), _lib.ptr(select), _lib.ptr(img),
                          _lib.ptr(fidx), *map(_lib.ptr, maps), _lib.ptr(ws))
        return img, fidx, maps

    def verts2uvimg(self, verts, cam):
        """verts [B,6890,3], cam [B,3] (s,tx,ty) -> IUV image [B,3,out,out] (renderer.py:256-278)."""
        return self._render(verts, cam)[0]

    def verts2maps(self, verts, cam):
        """Fused verts2uvimg + iuv_img2map (danet.py:165 -> 181-187): returns (iuv_image, [U,V,I,Ann])."""
        img, _, maps = self._render(verts, cam, want_maps=True)
        return img, maps

    def verts2faceidx(self, verts, cam):
        """Winning DensePose face id per pixel (-1 = background) -- the integer the parity tests pin."""
        img, fidx, _ = self._render(verts, cam, want_face_idx=True)
        return img, fidx

    def camera_matrix(self, cam):
        """renderer.py:280-298."""
        batch_size = cam.size(0)
        K = self.K.repeat(batch_size, 1, 1)
        R = self.R.repeat(batch_size, 1, 1)
        t = torch.stack([cam[:, 1], cam[:, 2], 2 * self.focal_length / (self.orig_size * cam[:, 0] + 1e-9)], dim=-1)
        t = t.unsqueeze(1)
        if cam.is_cuda:
            K, R, t = K.to(cam.device), R.to(cam.device), t.to(cam.device)
        return K, R, t
