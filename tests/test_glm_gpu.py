"""GPU: the interleaved rotary (B2_ROPE_INTERLEAVED, GLM's half_inner pairs).  The span-cache append with the interleaved
pairing equals the NeoX append of the dim-permuted rows bit for bit (q_out, 16-bit span rows, quantized codes after P^-1 and
{zero, scale}) over every step form, KV mode, FT, frequency form and rotary width; with the Q/K norm it equals b2_qk_rmsnorm
followed by the append without the norm; b2_rotary / b2_rotary_table satisfy the same identity and meet the fp64 GLM bound
at positions up to 131072, as the restated reference kernel does; the RotaryMulQuery operator (tests/glm_ref.py)."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import glm_ref as R
import glue_ref as G

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NH, NG, SPAN = 4, 2, 16
SLOTS = NH + 2 * NG
FORMS = {"single": (1, None), "chain2": (2, None), "chain7": (7, None), "chain16": (16, None),
         "tree": (6, [0, 0, 0, 1, 1, 3])}  # q_len, parents (depths 0, 1, 1, 2, 2, 3)
POS = [0, 1, 15, 16, 127, 4095, 32767, 131056]
BASE = 1e4
EPS = 1e-6


class _Pages:
    """Span tables for appends at far positions without a whole cache: each span a row lands in gets its own page, every
    other entry points at one shared guard page; every page starts 0xFF.  raw(): the stored row (codes unpacked to one value
    per dim) and its {zero, scale} bytes."""

    def __init__(self, slots, mode, dt):
        from b200spark import _lib
        qm = {"none": _lib.KV_NONE, "i8": _lib.KV_I8, "u4": _lib.KV_U4, "fp8": _lib.KV_FP8}[mode]
        max_spans = max(max(s) for s in slots) // SPAN + 1
        self.cfg = _lib.SpanCfg({torch.bfloat16: _lib.DT_BF16, torch.float16: _lib.DT_F16}[dt], qm, NH, NG, 128, SPAN, max_spans, 0)
        self.span_bytes = _lib.lib.b2_span_bytes(C.byref(self.cfg))
        self.stride = (self.span_bytes + 255) // 256 * 256
        self.mode, self.page = mode, {}
        self.row = {"none": 256, "i8": 128, "fp8": 128, "u4": 64}[mode]
        for b, ss in enumerate(slots):
            for s in ss:
                self.page.setdefault((b, s // SPAN), 1 + len(self.page))
        n = 1 + len(self.page)
        self.pools, tabs = {}, {}
        for which in "kv":
            pool = torch.full((n * self.stride,), 0xFF, dtype=torch.uint8, device="cuda")
            tab = torch.full((len(slots), max_spans), pool.data_ptr(), dtype=torch.int64)
            for (b, si), pg in self.page.items():
                tab[b, si] = pool.data_ptr() + pg * self.stride
            self.pools[which], tabs[which] = pool, tab.cuda()
        self.k_tab, self.v_tab = tabs["k"], tabs["v"]

    def raw(self, which, b, s):
        """(values [NG, 128] as int64 codes / 16-bit patterns, params bytes [NG, 8] or None) of slot s of sequence b"""
        pool = self.pools[which].cpu().numpy()
        off = self.page[(b, s // SPAN)] * self.stride
        n_rows = NG * SPAN
        rows = pool[off:off + n_rows * self.row].reshape(NG, SPAN, self.row)[:, s % SPAN]
        if self.mode == "none":
            vals = rows.view(np.uint16).astype(np.int64)
        elif self.mode == "u4":
            vals = np.stack([rows & 0xF, rows >> 4], -1).reshape(NG, 128).astype(np.int64)  # even dim in the low nibble
        else:
            vals = rows.astype(np.int64)
        prm = None
        if self.mode != "none":
            prm = pool[off + n_rows * self.row:off + n_rows * (self.row + 8)].reshape(NG, SPAN, 8)[:, s % SPAN]
        return vals, prm


def _bits(t):
    return t.contiguous().view(torch.int16).cpu().numpy()


def _step(form, ft, seed):
    q_len, parents = FORMS[form]
    rng = np.random.default_rng(seed)
    x = G.ft_values(rng.standard_normal((len(POS) * q_len, SLOTS, 128)) * 2, ft)
    kw = {} if q_len == 1 else {"q_len": q_len}
    if parents:
        kw["parents"] = torch.tensor([parents] * len(POS), dtype=torch.int32, device="cuda")
    slots = [[p + t for t in range(q_len)] for p in POS]
    return x, kw, slots


def _rope(freq, rd, style):
    """the rope tuple of ops._cache_append: computed frequencies at BASE, or the same base frequencies as a table"""
    from b200spark import ops
    if freq == "computed":
        return (BASE, rd, style)
    inv, af = ops.rope_table(None, BASE, rd, "cuda")
    return (inv, af, style)


@pytest.mark.parametrize("ft", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("mode", ["none", "i8", "u4", "fp8"])
def test_append_interleaved_equals_neox_of_permuted_rows(mode, ft):
    from b200spark import ops
    n_checked = 0
    for fi, form in enumerate(FORMS):
        for freq in ("computed", "table"):
            for rd in (64, 128):
                x, kw, slots = _step(form, ft, 100 * fi + rd)
                rows = x.shape[0]
                xi = G.to_ft(x.reshape(rows, -1), ft).cuda()
                xn = G.to_ft(R.apply_p(x, rd).reshape(rows, -1), ft).cuda()
                old = torch.tensor(POS, dtype=torch.int32, device="cuda")
                il, nx = _Pages(slots, mode, ft), _Pages(slots, mode, ft)
                q_il = ops._cache_append(il, xi, old, rope=_rope(freq, rd, "interleaved"), **kw)
                q_nx = ops._cache_append(nx, xn, old, rope=_rope(freq, rd, "neox"), **kw)
                torch.cuda.synchronize()
                tag = (form, freq, rd)
                qa = _bits(q_il).reshape(rows, NH, 128)
                qb = R.apply_p_inv(_bits(q_nx).reshape(rows, NH, 128), rd)
                assert np.array_equal(qa, qb), tag
                # the rotary did something: the interleaved rows differ from the NeoX append of the unpermuted rows
                q_plain = ops._cache_append(_Pages(slots, mode, ft), xi, old, rope=_rope(freq, rd, "neox"), **kw)
                assert not torch.equal(q_plain, q_il), tag
                for b, ss in enumerate(slots):
                    for s in ss:
                        for which in "kv":
                            va, pa = il.raw(which, b, s)
                            vb, pb = nx.raw(which, b, s)
                            assert np.array_equal(va, R.apply_p_inv(vb, rd)), tag + (which, b, s)
                            if pa is not None:
                                assert np.array_equal(pa, pb), tag + (which, b, s)
                            n_checked += 1
                # the guard pages were not written
                for which in "kv":
                    assert bool((il.pools[which][:il.stride] == 0xFF).all()), tag
    assert n_checked == 2 * 2 * 2 * len(POS) * sum(q for q, _ in FORMS.values())


@pytest.mark.parametrize("ft", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
def test_append_with_qk_norm_equals_norm_then_append(ft):
    """the fused norm + interleaved rotary equals b2_qk_rmsnorm followed by the interleaved append without the norm: every
    page byte and q_out"""
    from b200spark import ops
    g = torch.Generator(device="cuda").manual_seed(3)
    norm = tuple((1 + 0.1 * torch.randn(128, generator=g, device="cuda")).to(ft) for _ in range(2)) + (EPS,)
    for mode in ("none", "i8", "u4", "fp8"):
        for fi, form in enumerate(FORMS):
            for freq in ("computed", "table"):
                rd = 64 if fi % 2 else 128
                x, kw, slots = _step(form, ft, 7 * fi + 1)
                rows = x.shape[0]
                xd = G.to_ft(x.reshape(rows, -1), ft).cuda()
                old = torch.tensor(POS, dtype=torch.int32, device="cuda")
                rope = _rope(freq, rd, "interleaved")
                fused, comp = _Pages(slots, mode, ft), _Pages(slots, mode, ft)
                qf = ops._cache_append(fused, xd, old, rope=rope, qk_norm=norm, **kw)
                y = ops.qk_rmsnorm(xd, NH, NG, norm[0], norm[1], EPS)
                qc = ops._cache_append(comp, y, old, rope=rope, **kw)
                torch.cuda.synchronize()
                tag = (mode, form, freq)
                assert torch.equal(_bits_t(qf), _bits_t(qc)), tag
                for which in "kv":
                    assert torch.equal(fused.pools[which], comp.pools[which]), tag + (which,)


def _bits_t(t):
    return t.contiguous().view(torch.int16)


def test_standalone_rotary_identity_and_bound():
    """b2_rotary (bf16) and b2_rotary_table (bf16, fp16) with the interleaved pairing: NeoX of P x permuted back, bit for
    bit; the result and the restated reference kernel both within the fp64 GLM bound at positions up to 131072"""
    from b200spark import ops
    pos = np.array(G.ROPE_POS + [131072])
    rng = np.random.default_rng(11)
    pos_d = torch.tensor(pos, dtype=torch.int32, device="cuda")
    for ft in (torch.bfloat16, torch.float16):
        x = G.ft_values(rng.standard_normal((len(pos), SLOTS, 128)) * 2, ft)
        for rd in (64, 128):
            forms = [("table", invt, ratio) for invt in (1, 2) for ratio in (1.0, 500.0)]
            if ft == torch.bfloat16:
                forms.append(("computed", 2, 1.0))
            for kind, invt, ratio in forms:
                inv = torch.from_numpy(R.invfreq(invt, BASE, ratio, rd)).cuda()
                run = lambda rows, style: ops.rotary(rows, pos_d, NH, NG, base=BASE, rotary_dim=rd, style=style,
                                                     table=(inv, 1.0) if kind == "table" else None)
                yi = G.to_ft(x.reshape(len(pos), -1), ft).cuda()
                yn = G.to_ft(R.apply_p(x, rd).reshape(len(pos), -1), ft).cuda()
                run(yi, "interleaved")
                run(yn, "neox")
                torch.cuda.synchronize()
                tag = (str(ft), rd, kind, invt, ratio)
                a = _bits(yi).reshape(len(pos), SLOTS, 128)
                b = R.apply_p_inv(_bits(yn).reshape(len(pos), SLOTS, 128), rd)
                assert np.array_equal(a, b), tag
                y = yi.float().cpu().numpy().reshape(len(pos), SLOTS, 128)
                assert np.array_equal(y[:, NH + NG:], x[:, NH + NG:]), tag  # V heads untouched
                qk = x[:, :NH + NG]
                Y, D = R.glm64(qk, pos[:, None], R.theta64(invt, BASE, ratio, rd), rd)
                assert G.rope_ratio(y[:, :NH + NG], Y, D, ft).max() <= 1.0, tag
                if rd == 64:  # the reference kernel's own width: half the head
                    yr = R.half_inner32(qk, pos[:, None], R.invfreq(invt, BASE, ratio, rd), ft)
                    assert G.rope_ratio(yr, Y, D, ft).max() <= 1.0, tag


HOST_LIB = os.path.join(ROOT, "dash-infer_b200", "lib", "liballspark_b200.so")


def _host():
    import b200spark  # noqa: F401  (loads libb200spark.so with RTLD_GLOBAL first)
    lib = C.CDLL(HOST_LIB)
    lib.as_test_rotary_mulquery.restype = C.c_int
    lib.as_test_rotary_mulquery.argtypes = [C.c_int] * 6 + [C.c_float, C.c_float, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.as_test_set_dtype.restype = C.c_int
    lib.as_test_set_dtype.argtypes = [C.c_int]
    lib.as_test_registered.restype = C.c_int
    lib.as_test_registered.argtypes = [C.c_char_p]
    return lib


def _op(lib, x, ft, nH, nG, rtype, invt, ratio, pos):
    B = x.shape[0]
    xin = G.to_ft(x.reshape(B, -1), ft).contiguous()
    out = torch.empty_like(xin)
    p = np.asarray(pos, np.int32)
    st = lib.as_test_rotary_mulquery(B, nH, nG, nH * 128, rtype, invt, ratio, BASE, p.ctypes.data, xin.data_ptr(), out.data_ptr())
    return st, out


@pytest.mark.parametrize("ft", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
def test_rotary_mulquery_operator(ft):
    """type 3 against the restated reference kernel within the fp64 bound (invfreq_type 1 and 2, rope_ratio 1 and 500),
    and equal to b2_rotary_table with the same table; type 0 equals b2_rotary; other types are refused"""
    from b200spark import ops
    lib = _host()
    assert lib.as_test_registered(b"RotaryMulQuery") == 1
    assert lib.as_test_set_dtype({torch.bfloat16: 9, torch.float16: 2}[ft]) == 0
    try:
        nH, nG = 32, 2
        pos = np.array([0, 1, 17, 2047, 32768, 131072])
        rng = np.random.default_rng(5)
        x = G.ft_values(rng.standard_normal((len(pos), nH + 2 * nG, 128)) * 2, ft)
        for invt in (1, 2):
            for ratio in (1.0, 500.0):
                st, out = _op(lib, x, ft, nH, nG, 3, invt, ratio, pos)
                assert st == 0, (invt, ratio, st)
                y = out.float().numpy().reshape(x.shape)
                qk = x[:, :nH + nG]
                Y, D = R.glm64(qk, pos[:, None], R.theta64(invt, BASE, ratio), 64)
                yr = R.half_inner32(qk, pos[:, None], R.invfreq(invt, BASE, ratio), ft)
                assert G.rope_ratio(y[:, :nH + nG], Y, D, ft).max() <= 1.0, (invt, ratio)
                assert G.rope_ratio(yr, Y, D, ft).max() <= 1.0, (invt, ratio)
                assert np.array_equal(y[:, nH + nG:], x[:, nH + nG:])
                # the operator's table is the fp64 formula rounded once: b2_rotary_table with that table gives its bytes
                yd = G.to_ft(x.reshape(len(pos), -1), ft).cuda()
                inv = torch.from_numpy(R.invfreq(invt, BASE, ratio)).cuda()
                ops.rotary(yd, torch.tensor(pos, dtype=torch.int32, device="cuda"), nH, nG, table=(inv, 1.0),
                           style="interleaved")
                assert torch.equal(_bits_t(yd.cpu()), _bits_t(out)), (invt, ratio)
        if ft == torch.bfloat16:
            st, out = _op(lib, x, ft, nH, nG, 0, 0, 1.0, pos)
            assert st == 0
            yd = G.to_ft(x.reshape(len(pos), -1), ft).cuda()
            ops.rotary(yd, torch.tensor(pos, dtype=torch.int32, device="cuda"), nH, nG, base=BASE, rotary_dim=128)
            assert torch.equal(_bits_t(yd.cpu()), _bits_t(out))
        for rtype, invt in ((1, 2), (2, 2), (4, 2), (3, 0), (3, 3)):
            st, _ = _op(lib, x, ft, nH, nG, rtype, invt, 1.0, pos)
            assert st == 2, (rtype, invt, st)  # ALLSPARK_PARAM_ERROR: the configuration is not supported
    finally:
        lib.as_test_set_dtype(9)
