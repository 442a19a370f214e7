"""Python binding of the whole-network C entry (include/danet_b200.h danet_net_*, csrc/net.cu): loads a network
program written by plan.Plan.export() / DaNet.export_program() and replays it without the Python plan.  This is what a
non-Python host does through the same C calls (INTEGRATION.md, examples/net_host.c); here it mainly serves the tests
that hold the C executor to the Python plan bit for bit (the plan launches through the same step decoder, one step at a
time, with danet_net_run_step)."""
import ctypes

import torch

from . import _lib

GRAPH = 1                                             # DANET_NET_GRAPH


class _DevView(object):
    """__cuda_array_interface__ carrier: a torch view of memory the program owns (no copy)."""

    def __init__(self, ptr, shape, typestr):
        self.__cuda_array_interface__ = {"shape": tuple(shape), "typestr": typestr, "data": (ptr, False), "version": 2}


class NetProgram(object):
    def __init__(self, program, device="cuda:0"):
        """program: bytes of a network program, or a path to one."""
        if not torch.cuda.is_available():
            raise RuntimeError("danet_b200: CUDA device required (there is no CPU fallback)")
        self.lib = _lib.load()
        self.device = torch.device(device)
        self.h = ctypes.c_void_p()
        with torch.cuda.device(self.device):
            if isinstance(program, (bytes, bytearray)):
                buf = ctypes.create_string_buffer(bytes(program), len(program))
                _lib.check(self.lib.danet_net_load(ctypes.cast(buf, ctypes.c_void_p), len(program), ctypes.byref(self.h)), "net_load")
            else:
                _lib.check(self.lib.danet_net_load_file(str(program).encode(), ctypes.byref(self.h)), "net_load_file")
        b = ctypes.c_int32()
        chw = (ctypes.c_int32 * 3)()
        no = ctypes.c_int32()
        ns = ctypes.c_int32()
        _lib.check(self.lib.danet_net_info(self.h, ctypes.addressof(b), ctypes.addressof(chw), ctypes.addressof(no), ctypes.addressof(ns)), "net_info")
        self.batch, self.chw, self.n_steps = b.value, tuple(chw), ns.value
        self.names = [self.lib.danet_net_output_name(self.h, i).decode() for i in range(no.value)]

    def infer(self, images, graph=True):
        """images [B,3,H,W] fp32 on the program's device; asynchronous on the current stream."""
        if tuple(images.shape) != (self.batch,) + self.chw:
            raise ValueError("program compiled for input %r, got %r" % ((self.batch,) + self.chw, tuple(images.shape)))
        images = images.detach().to(self.device, torch.float32).contiguous()
        with torch.cuda.device(self.device):
            _lib.check(self.lib.danet_net_infer(self.h, _lib.ptr(images), GRAPH if graph else 0, _lib.stream_ptr(self.device)), "net_infer")

    def infer_host(self, images_np, graph=False):
        import numpy as np
        x = np.ascontiguousarray(images_np, dtype=np.float32)
        if tuple(x.shape) != (self.batch,) + self.chw:
            raise ValueError("program compiled for input %r, got %r" % ((self.batch,) + self.chw, tuple(x.shape)))
        _lib.check(self.lib.danet_net_infer_host(self.h, x.ctypes.data_as(ctypes.c_void_p), GRAPH if graph else 0), "net_infer_host")

    def output(self, name):
        """torch VIEW of a named output (overwritten by the next infer)."""
        p = ctypes.c_void_p()
        n = ctypes.c_uint64()
        dims = (ctypes.c_int32 * 4)()
        eb = ctypes.c_int32()
        _lib.check(self.lib.danet_net_output(self.h, name.encode(), ctypes.byref(p), ctypes.byref(n), ctypes.addressof(dims),
                                             ctypes.addressof(eb)), "net_output")
        shape = list(dims)                               # 4 dims, trailing ones for lower-rank outputs
        with torch.cuda.device(self.device):
            return torch.as_tensor(_DevView(p.value, shape, "<f4" if eb.value == 4 else "|u1"), device=self.device)

    def read_output(self, name):
        import numpy as np
        v = self.output(name)
        out = np.empty(tuple(v.shape), dtype=np.float32 if v.dtype == torch.float32 else np.uint8)
        _lib.check(self.lib.danet_net_read_output(self.h, name.encode(), out.ctypes.data_as(ctypes.c_void_p), out.nbytes), "net_read_output")
        return out

    def close(self):
        if self.__dict__.get("h") is not None and self.h:
            self.lib.danet_net_destroy(self.h)
            self.h = ctypes.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
