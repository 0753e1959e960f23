"""Register budget of the wgmma attention kernels (csrc/attn_tc.cu), read from the built library with
`cuobjdump -res-usage`: the forward kernel must fit two 288-thread CTAs per SM (<= 112 registers), and no attn_tc
kernel may spill to local memory.  Needs the CUDA toolkit's cuobjdump, not a GPU."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "vln-bevbert_b200", "libbevbert_b200.so")


def _cuobjdump():
    exe = shutil.which("cuobjdump")
    if exe is None:
        cand = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")
        exe = cand if os.path.exists(cand) else None
    return exe


def _attn_tc_usage():
    exe = _cuobjdump()
    if exe is None:
        pytest.skip("cuobjdump not found")
    assert os.path.exists(LIB), "%s not built" % LIB
    out = subprocess.run([exe, "-res-usage", LIB], check=True, capture_output=True, text=True).stdout
    usage = {}
    for m in re.finditer(r"Function (\S+):\s*\n\s*(.*)", out):
        name, fields = m.group(1), dict(re.findall(r"(\w+(?:\[\d+\])?):(\d+)", m.group(2)))
        if "attn_tc_" in name:
            usage[name] = {k: int(v) for k, v in fields.items()}
    return usage


def test_attn_tc_forward_fits_two_ctas_per_sm_and_nothing_spills():
    usage = _attn_tc_usage()
    fwd = [n for n in usage if "attn_tc_fwd_kernel" in n]
    bwd = [n for n in usage if "attn_tc_bwd_kernel" in n]
    assert len(fwd) == 1 and len(bwd) == 2, sorted(usage)
    # 2 CTAs x 288 threads x 112 registers = 64,512 <= 65,536
    assert usage[fwd[0]]["REG"] <= 112, usage[fwd[0]]
    for name, u in usage.items():
        assert u["STACK"] == 0 and u["LOCAL"] == 0, (name, u)
