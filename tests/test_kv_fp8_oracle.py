"""CPU: the fp8-e4m3 KV cache mode (B2_KV_FP8) — the CPU restatement of its quantizer, its span size and the argument
checks of the C ABI (no device needed)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
import torch

import kv_fp8_ref as F8
from oracle import kvcache_ref as KV

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _torch_quant(x):
    """Independent restatement in torch (elementwise fp32 tensor division, no division by a scalar)."""
    x = torch.from_numpy(x).float()
    amax = x.abs().amax(-1)
    scale = torch.clamp_min(amax, 1e-12) / torch.full_like(amax, 448.0)
    r = torch.ones_like(scale) / scale
    y = torch.clamp(x * r[..., None], -448.0, 448.0)
    return y.to(torch.float8_e4m3fn).view(torch.uint8).numpy(), scale.numpy()


@pytest.mark.parametrize("sigma", [1e-3, 1.0, 37.0])
def test_quantizer_against_torch_restatement(sigma):
    rng = np.random.default_rng(int(sigma * 1000))
    x = (rng.standard_normal((257, 128)) * sigma).astype(np.float32)
    x[3, 7] = 64 * sigma  # an outlier channel
    x[4] = 0.0            # an all-zero row: scale 1e-12 / 448, every code 0
    x = torch.from_numpy(x).to(torch.bfloat16).float().numpy()
    q, z, s = F8.quant_rows(x)
    tq, ts = _torch_quant(x)
    assert q.dtype == np.uint8 and np.array_equal(q, tq)
    assert np.array_equal(s, ts) and not z.any()
    assert not np.isin(q, [0x7F, 0xFF]).any()
    # relative precision of e4m3: 2^-4 at every magnitude above the subnormal range of the row
    xd = F8.dequant_rows(q, s)
    big = np.abs(x) >= s[:, None] * 2.0 ** -6
    assert np.all(np.abs(xd - x)[big] <= 2.0 ** -4 * np.abs(x)[big])


def test_quantizer_known_codes():
    x = np.zeros((1, 128), np.float32)
    vals = [448.0, -448.0, 1.0, -1.0, 2.0 ** -9, 2.0 ** -10, 3 * 2.0 ** -10, 1.0625, 1.1875, -0.0]
    x[0, :len(vals)] = vals  # amax 448: scale 1, the codes are e4m3 of the values themselves
    q, _, s = F8.quant_rows(x)
    assert s[0] == 1.0
    # 448 = 0x7E; 1.0 = 0x38; 2^-9 = smallest subnormal 0x01; 2^-10 ties to even 0; 1.5 * 2^-9 ties to 2^-8 = 0x02;
    # 1.0625 = 1 + 2^-4 ties to even 1.0; 1.1875 ties to 1.25 = 0x3A; -0.0 keeps its sign
    assert q[0, :len(vals)].tolist() == [0x7E, 0xFE, 0x38, 0xB8, 0x01, 0x00, 0x02, 0x38, 0x3A, 0x80]
    # saturation: a row whose maximum is huge still gives finite codes
    y = np.full((1, 128), 3e38, np.float32)
    y[0, 1] = -3e38
    q, _, s = F8.quant_rows(y)
    assert np.isfinite(s).all() and set(q[0].tolist()) <= {0x7E, 0xFE}


def test_span_cache_mirror_round_trip():
    rng = np.random.default_rng(0)
    ref = F8.SpanCacheFp8Ref(16, 2)
    ref.add_sequence()
    rows = rng.standard_normal((40, 2, 128)).astype(np.float32)
    for t in range(40):
        ref.append(0, t, rows[t])
    assert len(ref.spans[0]) == 3 and ref.spans[0][0].size == F8.span_bytes(16, 2)
    d = ref.dense(0, 40)
    assert d.shape == (2, 40, 128)
    q, _, s = F8.quant_rows(rows)
    assert np.array_equal(d, F8.dequant_rows(q, s).transpose(1, 0, 2))


def test_span_bytes_equal_i8():
    from b200spark import _lib
    lib = _lib.lib
    for span in (16, 32, 64, 128):
        for nG in (1, 4, 8):
            f8 = _lib.SpanCfg(_lib.DT_BF16, _lib.KV_FP8, 8 * nG, nG, 128, span, 16, 0)
            i8 = _lib.SpanCfg(_lib.DT_BF16, _lib.KV_I8, 8 * nG, nG, 128, span, 16, 0)
            nb = lib.b2_span_bytes(C.byref(f8))
            assert nb == lib.b2_span_bytes(C.byref(i8)) == F8.span_bytes(span, nG) == KV.span_bytes(KV.QUANT_I8, span, nG)
            assert lib.b2_span_attn_algo_bytes(C.byref(f8), 1000) == lib.b2_span_attn_algo_bytes(C.byref(i8), 1000) == 1000 * 2 * nG * 136
    f16 = _lib.SpanCfg(_lib.DT_F16, _lib.KV_FP8, 28, 4, 128, 128, 16, 0)
    assert lib.b2_span_bytes(C.byref(f16)) == F8.span_bytes(128, 4)
    # every mode: span bytes against the oracles; attention reads each token row of a span once (2 = K and V)
    oracle = {_lib.KV_NONE: lambda s, g: KV.span_bytes(KV.QUANT_NONE, s, g), _lib.KV_I8: lambda s, g: KV.span_bytes(KV.QUANT_I8, s, g),
              _lib.KV_U4: lambda s, g: KV.span_bytes(KV.QUANT_U4, s, g), _lib.KV_FP8: F8.span_bytes}
    for mode, ref in oracle.items():
        for span in (16, 32, 64, 128):
            for nG in (1, 2, 4, 8):
                cfg = _lib.SpanCfg(_lib.DT_BF16, mode, 8 * nG, nG, 128, span, 16, 0)
                assert lib.b2_span_bytes(C.byref(cfg)) == ref(span, nG)
                assert lib.b2_span_attn_algo_bytes(C.byref(cfg), 1000) == 1000 * 2 * ref(span, nG) // span


def test_header_value_matches_python(tmp_path):
    import b200spark
    from b200spark import _lib, model
    src = tmp_path / "v.c"
    src.write_text("#include <stdio.h>\n#include \"b200spark.h\"\nint main(void) { printf(\"%d\\n\", (int)B2_KV_FP8); return 0; }\n")
    exe = tmp_path / "v"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    out = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout
    assert int(out) == _lib.KV_FP8 == b200spark.KV_FP8 == F8.QUANT_FP8 == model.KV_MODES["fp8"] == 3


def test_rejected_configurations():
    """Head 64 with an fp8 cache is unsupported; modes above B2_KV_FP8 are parameter errors.  Both are caught by the
    argument checks, before any device work."""
    from b200spark import _lib
    lib = _lib.lib
    h = C.c_void_p()
    for ft in (_lib.DT_BF16, _lib.DT_F16):
        c64 = _lib.SpanCfg(ft, _lib.KV_FP8, 14, 2, 64, 16, 16, 0)
        assert lib.b2_span_bytes(C.byref(c64)) == 0
        assert lib.b2_span_attn_create(C.byref(h), C.byref(c64), 4) == 6
        assert lib.b2_span_cache_append(C.byref(c64), 1, 1, 1, 1, 1, 1, None, None) == 6
        assert lib.b2_span_context_copy(C.byref(c64), 1, 1, 256, 1, None) == 6
    bad = _lib.SpanCfg(_lib.DT_BF16, _lib.KV_FP8 + 1, 28, 4, 128, 16, 16, 0)
    assert lib.b2_span_bytes(C.byref(bad)) == 0
    assert lib.b2_span_attn_create(C.byref(h), C.byref(bad), 4) == 3
