"""ptxas report of the wgmma convolution engine (csrc/conv_tc.cu), compiled for sm_90a with the build's flags.

The engine is fast only while every warpgroup keeps several wgmma instructions in flight.  ptxas silently
serialises them (each MMA waits for the previous one) when an accumulator register is touched between them, when
the registers do not fit, or when a branch it cannot prove warp-uniform sits in the pipeline; it says so with an
info message C75xx "... serialized ..." (C7510-C7520).  Spilled accumulators have the same effect.  No GPU needed."""
import os
import re
import shutil
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


@pytest.fixture(scope="module")
def ptxas_log(tmp_path_factory):
    import __graft_entry__ as ge
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not os.path.exists(nvcc):
        nvcc = shutil.which("nvcc")
    if not nvcc:
        pytest.skip("nvcc not available")
    flags = [f for f in ge.NVCC_FLAGS if not f.startswith("--use_fast_math")]
    out = str(tmp_path_factory.mktemp("conv_tc_ptxas") / "conv_tc.o")
    r = subprocess.run([nvcc] + flags + ["-Xptxas", "-v", "-c", os.path.join(ge.CSRC, "conv_tc.cu"), "-o", out],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    return r.stdout + r.stderr


def _conv_kernels(log):
    """{mangled name of every k_conv_tc instantiation: (spill store bytes, spill load bytes)}"""
    res = {}
    for m in re.finditer(r"Function properties for (\S*k_conv_tc\S*)\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                         r"(\d+) bytes spill loads", log):
        res[m.group(1)] = (int(m.group(3)), int(m.group(4)))
    return res


def test_conv_tc_wgmma_not_serialized(ptxas_log):
    kernels = _conv_kernels(ptxas_log)
    assert len(kernels) == 2, kernels                     # k_conv_tc_fast and k_conv_tc_exact
    bad = [ln for ln in ptxas_log.splitlines() if re.search(r"\(C75\d\d\)", ln) and "serialized" in ln and "k_conv_tc" in ln]
    assert not bad, "\n".join(bad)


def test_conv_tc_no_spills(ptxas_log):
    kernels = _conv_kernels(ptxas_log)
    assert len(kernels) == 2, kernels
    for name, (st, ld) in kernels.items():
        assert st == 0 and ld == 0, "%s spills %d B stores / %d B loads" % (name, st, ld)
