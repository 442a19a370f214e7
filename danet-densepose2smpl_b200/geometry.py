"""utils/geometry.py of the reference, CUDA-backed (csrc/lbs.cu, csrc/targets.cu): rot6d_to_rotmat (:47-61),
batch_rodrigues / quat route (:9-45), perspective_projection (:63-91), estimate_translation (:94-157)."""
import torch

from . import _args, _lib


def _prep(x, name):
    _lib.require_cuda(x, name)
    return x.detach().float().contiguous()


@torch.no_grad()
def rot6d_to_rotmat(x):
    """(B,6)-like -> (B,3,3); input is viewed as (-1,3,2) exactly like the reference."""
    xc = _prep(x, "x").reshape(-1, 6)
    n = xc.shape[0]
    out = torch.empty(n, 3, 3, device=xc.device)
    with torch.cuda.device(xc.device):
        _lib.call("rot6d_to_rotmat", n, _lib.ptr(xc), _lib.ptr(out))
    return out


@torch.no_grad()
def batch_rodrigues(theta, flavor="quat"):
    """theta [B,3] axis-angle -> [B,3,3].  flavor 'quat' = utils/geometry.py:9-45; 'smplx' =
    smplx.lbs.batch_rodrigues (what pose2rot=True uses)."""
    tc = _prep(theta, "theta").reshape(-1, 3)
    n = tc.shape[0]
    out = torch.empty(n, 3, 3, device=tc.device)
    with torch.cuda.device(tc.device):
        _lib.call("batch_rodrigues", n, _lib.ptr(tc), _lib.ptr(out), 1 if flavor == "smplx" else 0)
    return out


@torch.no_grad()
def perspective_projection(points, rotation, translation, focal_length, camera_center):
    """points [B,N,3], rotation [B,3,3], translation [B,3], focal_length [B] or scalar,
    camera_center [B,2] -> [B,N,2]."""
    p = _prep(points, "points")
    B, N = p.shape[0], p.shape[1]
    dev = p.device
    r = rotation.detach().to(dev).float().contiguous()
    t = translation.detach().to(dev).float().contiguous()
    f = focal_length if torch.is_tensor(focal_length) else torch.full((B,), float(focal_length))
    f = f.detach().to(dev).float().reshape(-1).expand(B).contiguous()
    c = camera_center.detach().to(dev).float().contiguous()
    out = torch.empty(B, N, 2, device=dev)
    with torch.cuda.device(dev):
        _lib.call("perspective_projection", B, N, _lib.ptr(p), _lib.ptr(r), _lib.ptr(t), _lib.ptr(f), _lib.ptr(c),
                  _lib.ptr(out))
    return out


@torch.no_grad()
def estimate_translation(S, joints_2d, focal_length=5000., img_size=224.):
    """utils/geometry.py:135-157 on the device, with no host round trip: S [B,49,3] joints, joints_2d [B,49,3] key points
    (x, y in pixels, confidence); joints 25..48 are used -> the camera translation [B,3] (fp32, on S's device).
    The arithmetic is the reference's: fp32 sqrt(confidence) weights, the normal equations and their LU solve in fp64,
    one rounding to fp32.  Where numpy would raise LinAlgError (a singular system: every confidence 0), the row is NaN;
    negative confidences and non-finite joints give NaN as well."""
    where = "danet_b200.geometry.estimate_translation"
    _args.tensor(where, "S", S, dim=3)
    B = S.shape[0]
    _args.tensor(where, "S", S, shape=(B, 49, 3))
    _args.tensor(where, "joints_2d", joints_2d, shape=(B, 49, 3))
    f = _args.number(where, "focal_length", focal_length)
    size = _args.number(where, "img_size", img_size)
    _args.cuda(where, [("S", S), ("joints_2d", joints_2d)])
    out = torch.empty(B, 3, device=S.device)
    if B == 0:
        return out
    with torch.cuda.device(S.device):
        _lib.call("estimate_translation", B, _lib.ptr(S), _lib.ptr(joints_2d), f, size, _lib.ptr(out), device=S.device)
    return out
