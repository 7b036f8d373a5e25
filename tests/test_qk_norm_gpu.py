"""GPU: the per-head Q/K RMSNorm (QKLayerNormNoBeta).  The stand-alone b2_qk_rmsnorm against the restatement on exact
inputs and against the fp64 envelope on realistic rows (tests/qk_norm_ref.py); the fused norm of
b2_span_cache_append_qknorm against b2_qk_rmsnorm followed by the append without the norm, bit for bit, over every KV mode,
FT, step form, span length, rotary width and head layout; the QKLayerNormNoBeta operator against b2_qk_rmsnorm."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import glue_ref as G
import qk_norm_ref as R

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DTS = {"bf16": torch.bfloat16, "fp16": torch.float16}
EPS = 1e-6


def _t(x, dt):
    return torch.from_numpy(np.ascontiguousarray(x, np.float32)).to(dt).cuda()


def _np(t):
    return t.float().cpu().numpy().astype(np.float64)


@pytest.mark.parametrize("dt", ["bf16", "fp16"])
def test_standalone_exact_inputs(dt):
    """every head row equals the restatement for one rs candidate; out of place into a strided buffer with guard columns and
    rows left untouched, and in place with the same bytes"""
    from b200spark import ops
    ft = DTS[dt]
    rng = np.random.default_rng(3)
    nH, nG, rows = 4, 2, 48
    W = (nH + 2 * nG) * 128
    x, g = R.exact_batch(rows * (nH + 2 * nG), ft, rng)
    _, kg = R.exact_batch(1, ft, rng)
    x = x.reshape(rows, W)
    ld = W + 64
    guard = torch.full((rows + 2, ld), -7.0, dtype=ft, device="cuda")
    xs = guard.clone()
    xs[1:-1, :W] = _t(x, ft)
    xin = xs[1:-1, :W]
    out = guard.clone()
    y = ops.qk_rmsnorm(xin, nH, nG, _t(g, ft), _t(kg, ft), EPS, out=out[1:-1, :W])
    torch.cuda.synchronize()
    assert torch.equal(out[0], guard[0]) and torch.equal(out[-1], guard[-1]) and torch.equal(out[:, W:], guard[:, W:])
    yv = _np(y).reshape(rows, nH + 2 * nG, 128)
    xh = x.reshape(rows, nH + 2 * nG, 128)
    for j in range(nH + nG):
        bad = R.exact_rows_failing(yv[:, j], xh[:, j], g if j < nH else kg, EPS, ft)
        assert len(bad) == 0, (j, bad[:4])
    assert np.array_equal(yv[:, nH + nG:], xh[:, nH + nG:])  # V copied
    before = xs.clone()
    ops.qk_rmsnorm(xin, nH, nG, _t(g, ft), _t(kg, ft), EPS, out=xin)  # in place
    torch.cuda.synchronize()
    assert torch.equal(xin, y)
    assert torch.equal(xs[0], before[0]) and torch.equal(xs[:, W:], before[:, W:])


@pytest.mark.parametrize("dt", ["bf16", "fp16"])
@pytest.mark.parametrize("kind", R.ROW_KINDS)
def test_standalone_realistic_rows(dt, kind):
    """N(0,1) rows and rows with a 64-sigma channel, per-row RMS 2^-12 .. 2^12 (fp16: while the rows stay finite), inside
    the fp64 envelope"""
    from b200spark import ops
    ft = DTS[dt]
    rng = np.random.default_rng(11)
    nH, nG = 8, 1
    qg, kg = R.gammas(ft, rng)
    top = 12 if ft == torch.bfloat16 else (9 if kind == "spike" else 12)
    worst = 0.0
    for s in range(-12, top + 1, 3):
        x = R.realistic_rows(32, (nH + 2 * nG) * 128, ft, rng, kind, s)
        y = _np(ops.qk_rmsnorm(_t(x, ft), nH, nG, _t(qg, ft), _t(kg, ft), EPS))
        worst = max(worst, float(R.ratio(y, R.exact(x, nH, nG, qg, kg, EPS), ft).max()))
    assert worst <= 1.0, worst


def test_standalone_error_codes_and_graph_replay():
    from b200spark import _lib, ops
    lib = _lib.lib
    x = torch.randn(4, 6 * 128, device="cuda").to(torch.bfloat16)
    g = torch.ones(128, dtype=torch.bfloat16, device="cuda")
    nrm = _lib.QkNorm(g.data_ptr(), g.data_ptr(), EPS, 0)
    p = C.c_void_p(x.data_ptr())
    assert lib.b2_qk_rmsnorm(p, p, 4, 768, 4, 1, 128, None, _lib.DT_BF16, None) == 3
    assert lib.b2_qk_rmsnorm(p, p, 4, 640, 4, 1, 128, C.byref(nrm), _lib.DT_BF16, None) == 3
    assert lib.b2_qk_rmsnorm(p, p, 4, 768, 4, 1, 64, C.byref(nrm), _lib.DT_BF16, None) == 6
    assert lib.b2_qk_rmsnorm(C.c_void_p(x.data_ptr() + 2), p, 3, 768, 4, 1, 128, C.byref(nrm), _lib.DT_BF16, None) == 6
    bad = _lib.QkNorm(g.data_ptr() + 2, g.data_ptr(), EPS, 0)
    assert lib.b2_qk_rmsnorm(p, p, 4, 768, 4, 1, 128, C.byref(bad), _lib.DT_BF16, None) == 6
    with pytest.raises(AssertionError):
        ops.qk_rmsnorm(x, 4, 1, g.float(), g, EPS)  # gamma dtype must be the model's
    # CUDA graph: the replay writes what the eager call wrote
    qg = (1 + 0.1 * torch.randn(128, device="cuda")).to(torch.bfloat16)
    y0 = ops.qk_rmsnorm(x, 4, 1, qg, g, EPS)
    y = torch.empty_like(x)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        ops.qk_rmsnorm(x, 4, 1, qg, g, EPS, out=y)
        gr = torch.cuda.CUDAGraph()
        with torch.cuda.graph(gr, stream=s):
            ops.qk_rmsnorm(x, 4, 1, qg, g, EPS, out=y)
    torch.cuda.synchronize()
    y.zero_()
    gr.replay()
    torch.cuda.synchronize()
    assert torch.equal(y, y0)


# ------------------------------------------------------------------------------------------------ fused = composed
MODES = ["none", "i8", "u4", "fp8"]
LAYOUTS = [(32, 8), (16, 8), (8, 1), (16, 1)]
FORMS = {"single": 1, "chain": 3, "tree": 5}


def _mode(m):
    from b200spark import _lib
    return {"none": _lib.KV_NONE, "i8": _lib.KV_I8, "u4": _lib.KV_U4, "fp8": _lib.KV_FP8}[m]


def _append_pair(mode, ft, form, span, rdim, nH, nG, B, seed, graph=False):
    """(composed caches + q, fused caches + q) for one step of B sequences"""
    from b200spark import ops
    T = FORMS[form]
    g = torch.Generator(device="cuda").manual_seed(seed)
    qkv = torch.randn(B * T, (nH + 2 * nG) * 128, generator=g, device="cuda").mul_(2.0).to(ft)
    qg = (1 + 0.1 * torch.randn(128, generator=g, device="cuda")).to(ft)
    kg = (1 + 0.1 * torch.randn(128, generator=g, device="cuda")).to(ft)
    old = torch.tensor([(7 * b + 3) % 40 for b in range(B)], dtype=torch.int32, device="cuda")
    kw = {} if form == "single" else {"q_len": T}
    if form == "tree":
        kw["parents"] = torch.tensor([[0, 0, 0, 1, 1], [0, 0, 1, 2, 0]] * (B // 2) + [[0, 0, 1, 1, 3]] * (B % 2),
                                     dtype=torch.int32, device="cuda")
    rope = (1e6, rdim)
    mk = lambda: ops.SpanCache(B, 64, nH, nG, span, _mode(mode), fill=0xFF, dtype=ft)
    ca, cb = mk(), mk()
    qn = ops.qk_rmsnorm(qkv, nH, nG, qg, kg, EPS)
    qa = ops._cache_append(ca, qn, old, rope=rope, **kw)
    if not graph:
        qb = ops._cache_append(cb, qkv, old, rope=rope, qk_norm=(qg, kg, EPS), **kw)
    else:
        qb = torch.empty_like(qa)
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            gr = torch.cuda.CUDAGraph()
            with torch.cuda.graph(gr, stream=s):
                ops._cache_append(cb, qkv, old, q_out=qb, rope=rope, qk_norm=(qg, kg, EPS), **kw)
        torch.cuda.synchronize()
        gr.replay()
    torch.cuda.synchronize()
    return (ca, qa), (cb, qb)


def _same(a, b):
    (ca, qa), (cb, qb) = a, b
    return torch.equal(ca.k_pool, cb.k_pool) and torch.equal(ca.v_pool, cb.v_pool) and torch.equal(qa, qb)


@pytest.mark.parametrize("form", list(FORMS))
@pytest.mark.parametrize("dt", ["bf16", "fp16"])
@pytest.mark.parametrize("mode", MODES)
def test_fused_equals_composed(mode, dt, form):
    """span bytes, {zero, scale} and q_out of the fused append equal b2_qk_rmsnorm + the append without the norm"""
    ft = DTS[dt]
    n = 0
    for span in (16, 128):
        for rdim in (128, 64):
            for nH, nG in LAYOUTS:
                a, b = _append_pair(mode, ft, form, span, rdim, nH, nG, 3, seed=n)
                assert _same(a, b), (span, rdim, nH, nG)
                n += 1


@pytest.mark.parametrize("form", list(FORMS))
def test_fused_repeat_and_graph_replay(form):
    a, b = _append_pair("i8", torch.bfloat16, form, 16, 128, 16, 8, 4, seed=5)
    a2, b2 = _append_pair("i8", torch.bfloat16, form, 16, 128, 16, 8, 4, seed=5)
    assert _same(a, b) and _same(a2, b2) and _same(b, b2)
    _, bg = _append_pair("i8", torch.bfloat16, form, 16, 128, 16, 8, 4, seed=5, graph=True)
    assert _same(b, bg)


def test_fused_q_len_limit():
    from b200spark import _lib, ops
    c = ops.SpanCache(1, 64, 8, 1, 16, _lib.KV_NONE)
    qkv = torch.zeros(17, 10 * 128, dtype=torch.bfloat16, device="cuda")
    g = torch.ones(128, dtype=torch.bfloat16, device="cuda")
    with pytest.raises(_lib.B2Error):
        ops._cache_append(c, qkv, torch.zeros(1, dtype=torch.int32, device="cuda"), q_len=17, qk_norm=(g, g, EPS))


# ------------------------------------------------------------------------------------------------ the C++ operator
def _host_lib():
    lib = C.CDLL(os.path.join(ROOT, "dash-infer_b200", "lib", "liballspark_b200.so"))
    lib.as_test_qk_layernorm.restype = C.c_int
    lib.as_test_qk_layernorm.argtypes = [C.c_int] * 5 + [C.c_float] + [C.c_void_p] * 4
    lib.as_test_set_dtype.restype = C.c_int
    lib.as_test_set_dtype.argtypes = [C.c_int]
    lib.as_test_registered.restype = C.c_int
    lib.as_test_registered.argtypes = [C.c_char_p]
    return lib


@pytest.mark.parametrize("dt", ["bf16", "fp16"])
@pytest.mark.parametrize("nranks,heads,groups", [(1, 32, 8), (2, 32, 8), (4, 16, 1), (2, 16, 8)])
def test_operator_matches_b2_qk_rmsnorm(dt, nranks, heads, groups):
    """QKLayerNormNoBeta with the whole model's head counts on one rank of nranks: num_heads / nranks q heads and
    multi_query_group_num / nranks kv heads (a group count of 1 stays 1)"""
    from b200spark import _lib, ops
    ft = DTS[dt]
    lib = _host_lib()
    assert lib.as_test_registered(b"QKLayerNormNoBeta") == 1
    assert lib.as_test_set_dtype(_lib.DT_F16 if ft == torch.float16 else _lib.DT_BF16) == 0
    try:
        nH, nG, B = heads // nranks, (groups // nranks if groups != 1 else 1), 5
        g = torch.Generator().manual_seed(nranks * 100 + heads)
        x = torch.randn(B, (nH + 2 * nG) * 128, generator=g).to(ft)
        qg = (1 + 0.1 * torch.randn(128, generator=g)).to(ft)
        kg = (1 + 0.1 * torch.randn(128, generator=g)).to(ft)
        out = torch.empty_like(x)
        rc = lib.as_test_qk_layernorm(nranks, B, heads, groups, 128, EPS, x.data_ptr(), qg.data_ptr(), kg.data_ptr(), out.data_ptr())
        assert rc == 0, rc
        ref = ops.qk_rmsnorm(x.cuda(), nH, nG, qg.cuda(), kg.cuda(), EPS).cpu()
        assert torch.equal(out, ref)
    finally:
        lib.as_test_set_dtype(_lib.DT_BF16)
