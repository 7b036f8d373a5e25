"""Machine code of the batch 17-64 wgmma GEMM (`wq_gemm_tc_kernel`), read from the built library with cuobjdump (no GPU).

The consumer loop only overlaps the dequantization of one 64-k tile with the MMAs of the previous one if ptxas keeps a
tile's MMAs in one asynchronous group: chained HGMMAs (QGMMAs for fp8) with the group's `gsb0` on the last one only, and
no empty placeholder HGMMA standing in for `wgmma.commit_group`.  A runtime choice of the MMA width inside the loop breaks both
without any change in the results, so only the code shows it.
"""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "dash-infer_b200", "lib", "libb200spark.so")
CUOBJDUMP = shutil.which("cuobjdump") or next(
    (p for p in ("/usr/local/cuda/bin/cuobjdump",) if os.path.exists(p)), None)

pytestmark = pytest.mark.skipif(CUOBJDUMP is None, reason="cuobjdump not found")

# template arguments <WBITS, MULTI, A8, GROUPED, H> of the mangled name
_ARGS = re.compile(r"wq_gemm_tc_kernelILi(\d+)ELb([01])ELb([01])ELb([01])ELb([01])EE")


def _kernel(name):
    m = _ARGS.search(name)
    return (int(m.group(1)),) + tuple(int(x) for x in m.groups()[1:]) if m else None


def _cuobjdump(flag):
    assert os.path.exists(LIB), "build the library first: python dash-infer_b200/build.py"
    return subprocess.run([CUOBJDUMP, flag, LIB], check=True, capture_output=True, text=True).stdout


def _sass_by_kernel():
    out, cur = {}, None
    for line in _cuobjdump("-sass").splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = _kernel(m.group(1))
            if cur is not None:
                out[cur] = []
        elif cur is not None and re.search(r"\b[HQ]GMMA\.", line):  # bf16 / fp16 and fp8 warpgroup MMAs
            out[cur].append(line)
    return out


def test_mmas_of_a_tile_form_one_group():
    kernels = _sass_by_kernel()
    assert len(kernels) >= 18, sorted(kernels)
    for k, mmas in sorted(kernels.items()):
        assert mmas, k
        placeholders = [h for h in mmas if re.search(r"RZ, gdesc\[URZ\]", h)]
        assert not placeholders, (k, placeholders[:2])
        gsb0 = [h for h in mmas if "gsb0" in h]
        assert len(gsb0) < len(mmas), (k, len(gsb0), len(mmas))


def test_no_local_memory():
    """Every instantiation keeps its state in registers: no stack frame, no spills."""
    usage, cur = {}, None
    for line in _cuobjdump("-res-usage").splitlines():
        m = re.match(r"\s*Function (\S+):", line)
        if m:
            cur = _kernel(m.group(1))
        elif cur is not None and "REG:" in line:
            usage[cur] = int(re.search(r"STACK:(\d+)", line).group(1))
            cur = None
    assert len(usage) >= 18, sorted(usage)
    for k, stack in sorted(usage.items()):
        assert stack == 0, (k, stack)
