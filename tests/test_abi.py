"""CPU: the C-ABI library loads without a GPU and exports every function include/b200spark.h declares."""
import ctypes
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    src = open(os.path.join(ROOT, "include", "b200spark.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(b2_[a-z0-9_]+)\s*\(", src)))


def test_header_symbols_exported():
    from b200spark import _lib
    syms = declared_symbols()
    assert len(syms) >= 20
    dll = ctypes.CDLL(_lib.LIB_PATH)
    missing = [s for s in syms if not hasattr(dll, s)]
    assert not missing, missing
    assert sorted(_lib.SYMBOLS) == syms, set(_lib.SYMBOLS) ^ set(syms)


def test_status_strings_and_version():
    from b200spark import lib
    assert lib.b2_status_string(0) == b"B2_OK"
    assert lib.b2_status_string(3) == b"B2_ERR_PARAM"
    assert b"sm_90a" in lib.b2_version()


def test_param_validation_without_gpu():
    """Calls that must fail on argument checks before touching the device."""
    import ctypes as C
    from b200spark import _lib
    lib = _lib.lib
    h = C.c_void_p()
    bad = _lib.GemmDesc(128, 128, 5, -1, _lib.DT_BF16, _lib.DT_U8, 8, 0)  # wbits 5
    assert lib.b2_gemm_wq_create(C.byref(h), C.byref(bad)) == 3
    bad = _lib.GemmDesc(128, 128, 4, -1, _lib.DT_F32, _lib.DT_U8, 8, 0)  # FT is bf16 or fp16; fp32 activations -> unsupported
    assert lib.b2_gemm_wq_create(C.byref(h), C.byref(bad)) == 6
    bad = _lib.GemmDesc(128, 128, 4, -1, _lib.DT_BF16, _lib.DT_I8, 8, 0)  # A16W4 is uint4x2 only (gemm_a16w4.cpp:104-110)
    assert lib.b2_gemm_wq_create(C.byref(h), C.byref(bad)) == 3
    cfg = _lib.SpanCfg(_lib.DT_BF16, 0, 28, 4, 64, 128, 16, 0)  # head 64 (config C0): bf16 KV only
    assert lib.b2_span_bytes(C.byref(cfg)) == 128 * 4 * 64 * 2
    cfg = _lib.SpanCfg(_lib.DT_BF16, 1, 28, 4, 64, 128, 16, 0)  # head 64 with quantized KV: unsupported (like the reference)
    assert lib.b2_span_bytes(C.byref(cfg)) == 0
    cfg = _lib.SpanCfg(_lib.DT_BF16, 0, 28, 4, 96, 128, 16, 0)
    assert lib.b2_span_bytes(C.byref(cfg)) == 0
    cfg = _lib.SpanCfg(_lib.DT_BF16, 1, 28, 4, 128, 128, 16, 0)
    assert lib.b2_span_bytes(C.byref(cfg)) == 128 * 4 * 128 + 2 * 128 * 4 * 4  # virtual_cache.cpp:214-220
    cfg = _lib.SpanCfg(_lib.DT_BF16, 2, 28, 4, 128, 32, 16, 0)
    assert lib.b2_span_bytes(C.byref(cfg)) == 32 * 4 * 64 + 2 * 32 * 4 * 4
    cfg = _lib.SpanCfg(_lib.DT_BF16, 0, 28, 4, 128, 48, 16, 0)  # span 48 invalid (span_cache_config.cpp:32-48)
    assert lib.b2_span_bytes(C.byref(cfg)) == 0


def test_struct_layouts_match_the_header(tmp_path):
    """The ctypes mirrors in b200spark/_lib.py against the C compiler's view of include/b200spark.h (sizeof / offsetof of
    every struct that crosses the C ABI by pointer)."""
    import ctypes as C
    import subprocess
    from b200spark import _lib
    structs = {"b2_gemm_wq_desc": _lib.GemmDesc, "b2_span_cfg": _lib.SpanCfg, "b2_rope_cfg": _lib.RopeCfg, "b2_gemm_fuse": _lib.GemmFuse}
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "b200spark.h"', 'int main(void) {']
    for cname, cls in structs.items():
        lines.append('  printf("%s %%zu\\n", sizeof(%s));' % (cname, cname))
        for fname, _ in cls._fields_:
            lines.append('  printf("%s.%s %%zu\\n", offsetof(%s, %s));' % (cname, fname, cname, fname))
    lines += ['  return 0;', '}']
    src = tmp_path / "layout.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    out = dict(l.split() for l in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.splitlines())
    for cname, cls in structs.items():
        assert int(out[cname]) == C.sizeof(cls), cname
        for fname, _ in cls._fields_:
            assert int(out["%s.%s" % (cname, fname)]) == getattr(cls, fname).offset, (cname, fname)
