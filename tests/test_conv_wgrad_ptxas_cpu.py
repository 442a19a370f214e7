"""ptxas report of the weight-gradient kernel (csrc/conv_wgrad.cu), compiled for sm_90a with the build's flags.

k_wgrad is fast only while its warpgroup keeps wgmma instructions in flight; ptxas serialises them silently apart from an
info message C75xx "... serialized ..." and spilled accumulators have the same effect.  No GPU needed."""
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
    out = str(tmp_path_factory.mktemp("conv_wgrad_ptxas") / "conv_wgrad.o")
    r = subprocess.run([nvcc] + flags + ["-Xptxas", "-v", "-c", os.path.join(ge.CSRC, "conv_wgrad.cu"), "-o", out],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    return r.stdout + r.stderr


def _kernels(log):
    """{mangled name of every kernel: (spill store bytes, spill load bytes)}"""
    return {m.group(1): (int(m.group(3)), int(m.group(4))) for m in re.finditer(
        r"Function properties for (\S+)\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", log)}


def test_wgrad_wgmma_not_serialized(ptxas_log):
    assert any("k_wgrad" in n for n in _kernels(ptxas_log))
    bad = [ln for ln in ptxas_log.splitlines() if re.search(r"\(C75\d\d\)", ln) and "serialized" in ln]
    assert not bad, "\n".join(bad)


def test_wgrad_no_spills(ptxas_log):
    kernels = _kernels(ptxas_log)
    assert kernels
    for name, (st, ld) in kernels.items():
        assert st == 0 and ld == 0, "%s spills %d B stores / %d B loads" % (name, st, ld)
