"""Machine code of the per-head Q/K RMSNorm kernels, read from the built library with cuobjdump (no GPU): the stand-alone
kernel keeps everything in registers, and the fused norm adds no local memory to the span-cache append."""
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

# cache_append_kernel<QM, H, MT, TREE, QKN>
_APPEND = re.compile(r"cache_append_kernelILi(\d)ELb([01])ELb([01])ELb([01])ELb([01])EE")


def _stacks():
    assert os.path.exists(LIB), "build the library first: python dash-infer_b200/build.py"
    out = subprocess.run([CUOBJDUMP, "-res-usage", LIB], check=True, capture_output=True, text=True).stdout
    usage, cur = {}, None
    for line in out.splitlines():
        m = re.match(r"\s*Function (\S+):", line)
        if m:
            cur = m.group(1)
        elif cur is not None and "REG:" in line:
            usage[cur] = int(re.search(r"STACK:(\d+)", line).group(1))
            cur = None
    return usage


def test_standalone_kernel_has_no_local_memory():
    usage = _stacks()
    qk = {n: s for n, s in usage.items() if "qk_rmsnorm_kernel" in n}
    assert len(qk) == 2, sorted(qk)
    assert all(s == 0 for s in qk.values()), qk


def test_fused_norm_adds_no_local_memory_to_the_append():
    """The appends without the norm already carry sincosf's slow-path range reduction in a 32-byte frame; the norm's
    instantiations keep that frame.  In the fp8 tree form ptxas saves one more register (8 bytes) across the call into
    that slow path, which the norm's extra live values cause; no instantiation spills the norm's own state."""
    usage = _stacks()
    append = {tuple(int(g) for g in _APPEND.search(n).groups()): s for n, s in usage.items() if _APPEND.search(n)}
    assert len(append) == 48, len(append)
    for k, s in sorted(append.items()):
        if k[4]:
            plain = append[k[:4] + (0,)]
            assert s <= plain + 8, (k, s, plain)
