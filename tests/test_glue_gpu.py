"""GPU: the decode step's glue kernels against exact references (tests/glue_ref.py) at their edges.

RMSNorm within half an FT ulp + the fp32 budget of exact, per element, and mostly equal to rn_FT(exact); rotary in all three
implementations (b2_rotary, the head-128 cache append in its single-token, chain and tree forms, the head-64 append)
against the kernels' formula and fp64 NeoX at positions up to 131071; argmax, the vocab-split shard + merge, binary,
embedding and lens_add bit-exact."""
import ctypes as C

import numpy as np
import pytest
import torch

import glue_ref as G

pytestmark = pytest.mark.gpu


def _np(t):
    return t.float().cpu().numpy()


# ---------------------------------------------------------------- RMSNorm
@pytest.mark.parametrize("cols", G.RMS_COLS)
@pytest.mark.parametrize("dt", ["bf16", "fp16"])
def test_rmsnorm(dt, cols):
    """every row kind (random, constant, one dominant element, all zero, eps-dominated, large up to sum(x^2) = 2^125) at
    1 / 3 / 64 / 130 rows, both eps; in place gives the same bits"""
    from b200spark import ops
    ft = G.FTS[dt]
    worst, miss, total = 0.0, 0, 0
    for rows in G.RMS_ROWS:
        x, g = G.rms_batch(rows, cols, ft, seed=rows * 100003 + cols)
        xd, gd = G.to_ft(x, ft).cuda(), G.to_ft(g, ft).cuda()
        for eps in G.RMS_EPS:
            y = ops.rmsnorm(xd, gd, eps)
            assert y.dtype == ft
            ratio, m, n = G.rms_check(_np(y), x, g, eps, ft)
            assert ratio <= 1.0, (rows, eps, ratio)
            assert m <= G.rms_allowed_mismatches(n), (rows, eps, m, n)
            worst, miss, total = max(worst, ratio), miss + m, total + n
            xi = xd.clone()
            ops.rmsnorm(xi, gd, eps, out=xi)
            assert torch.equal(xi.view(torch.int16), y.view(torch.int16)), (rows, eps)
    print("rmsnorm %s cols %5d: worst error/bound %.3f, %d of %d elements != rn(exact)" % (dt, cols, worst, miss, total))


# ---------------------------------------------------------------- rotary
NH, NG, SPAN = 4, 2, 16
ROPE_WORST = {}  # (impl, dt, rotary_dim, base, pos) -> (worst |y - NeoX64|, worst ratio to its bound)


def _rope_check(impl, got, x, pos, base, rd, dt):
    """got, x: [R, heads, head] values; pos: [R] rotary positions.  Both bounds per element, dims >= rd untouched."""
    pos = np.asarray(pos)
    Y, D = G.rope_formula(x, pos[:, None], base, rd)
    r = G.rope_ratio(got, Y, D, dt)
    i = np.unravel_index(int(np.argmax(r)), r.shape)
    assert r.max() <= 1.0, (impl, base, rd, "row %d head %d dim %d" % i, float(got[i]), float(Y[i]), int(pos[i[0]]))
    Y64, D64 = G.rope_neox64(x, pos[:, None], base, rd)
    r64 = G.rope_ratio(got, Y64, D64, dt)
    assert r64.max() <= 1.0, (impl, base, rd, float(r64.max()))
    assert np.array_equal(got[..., rd:], x[..., rd:]), impl
    err = np.abs(np.asarray(got, np.float64) - Y64)
    for p in np.unique(pos):
        k = (impl, str(dt).split(".")[-1], rd, base, int(p))
        e, q = float(err[pos == p].max()), float(r64[pos == p].max())
        a, b = ROPE_WORST.get(k, (0.0, 0.0))
        ROPE_WORST[k] = (max(a, e), max(b, q))


def _print_worst(impl, dt, rd):
    """one line per base: position: worst |y - NeoX64| (worst ratio to its bound)"""
    for key in sorted({k[1:4] for k in ROPE_WORST if k[:3] == (impl, str(dt).split(".")[-1], rd)}):
        cells = ["%d: %.2e (%.2f)" % ((p,) + ROPE_WORST[(impl,) + key + (p,)]) for p in G.ROPE_POS if (impl,) + key + (p,) in ROPE_WORST]
        print("rope vs fp64 %s %s rd %d base %.0e | %s" % ((impl,) + key + (" | ".join(cells),)))


class _Pages:
    """Span tables for appends at far positions without a whole cache: each span a row lands in gets its own page, every
    other table entry points at one shared guard page; every page starts 0xFF.  Duck-types ops.SpanCache for the appends."""

    def __init__(self, slots, nH, nG, head, dt):
        from b200spark import _lib
        self.dt, self.nG, self.head = dt, nG, head
        max_spans = max(max(s) for s in slots) // SPAN + 1
        self.cfg = _lib.SpanCfg({torch.bfloat16: _lib.DT_BF16, torch.float16: _lib.DT_F16}[dt], _lib.KV_NONE, nH, nG, head, SPAN,
                                max_spans, 0)
        self.span_bytes = _lib.lib.b2_span_bytes(C.byref(self.cfg))
        self.stride = (self.span_bytes + 255) // 256 * 256
        self.page = {}
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

    def rows(self, which, b, slots):
        """[len(slots), nG, head] values of the given slots of sequence b"""
        pool = self.pools[which].cpu()
        out = []
        for s in slots:
            off = self.page[(b, s // SPAN)] * self.stride
            out.append(pool[off:off + self.span_bytes].view(self.dt).reshape(self.nG, SPAN, self.head)[:, s % SPAN].float().numpy())
        return np.stack(out)

    def untouched(self, which, written):
        """every byte outside the written (b, slot) rows still 0xFF (the guard page included)"""
        pool = self.pools[which].cpu().numpy().copy()
        row = self.head * 2
        for b, s in written:
            off = self.page[(b, s // SPAN)] * self.stride
            for g in range(self.nG):
                r = off + (g * SPAN + s % SPAN) * row
                pool[r:r + row] = 0xFF
        return bool((pool == 0xFF).all())


def _qkv(R, heads, head, dt, seed):
    rng = np.random.default_rng(seed)
    return G.ft_values(rng.standard_normal((R, heads, head)) * 2, dt)


def _tree_depths(parents):
    d = [0] * len(parents)
    for t in range(1, len(parents)):
        d[t] = d[parents[t]] + 1
    return d


FORMS = {"single": (1, None), "tokens": (3, None), "tree": (4, [0, 0, 0, 1])}  # q_len, parents (depths 0, 1, 1, 2)


@pytest.mark.parametrize("form", list(FORMS))
@pytest.mark.parametrize("rd", [128, 64])
@pytest.mark.parametrize("dt", ["bf16", "fp16"])
def test_rope_append_head128(form, rd, dt):
    """The fused head-128 append: q_out and the K rows within both bounds at every position and base (a tree row carries
    the RoPE of old_len + depth), dims >= rotary_dim and the V rows keep their input bits, no other span byte changes."""
    from b200spark import ops
    ft = G.FTS[dt]
    q_len, parents = FORMS[form]
    B, slots_n = len(G.ROPE_POS), NH + 2 * NG
    depth = _tree_depths(parents) if parents else list(range(q_len))
    for base in G.ROPE_BASES:
        slots = [[p + t for t in range(q_len)] for p in G.ROPE_POS]
        cache = _Pages(slots, NH, NG, 128, ft)
        x = _qkv(B * q_len, slots_n, 128, ft, seed=rd + q_len)
        old = torch.tensor(G.ROPE_POS, dtype=torch.int32, device="cuda")
        xd = G.to_ft(x.reshape(B * q_len, -1), ft).cuda()
        kw = {} if q_len == 1 else {"q_len": q_len}
        if parents:
            kw["parents"] = torch.tensor([parents] * B, dtype=torch.int32, device="cuda")
        qo = ops._cache_append(cache, xd, old, rope=(base, rd), **kw)
        torch.cuda.synchronize()
        rpos = np.array([p + depth[t] for p in G.ROPE_POS for t in range(q_len)])
        name = "app128-" + form
        _rope_check(name, _np(qo).reshape(B * q_len, NH, 128), x[:, :NH], rpos, base, rd, ft)
        k = np.concatenate([cache.rows("k", b, slots[b]) for b in range(B)])
        v = np.concatenate([cache.rows("v", b, slots[b]) for b in range(B)])
        _rope_check(name, k, x[:, NH:NH + NG], rpos, base, rd, ft)
        assert np.array_equal(v, x[:, NH + NG:])
        written = [(b, s) for b in range(B) for s in slots[b]]
        assert cache.untouched("k", written) and cache.untouched("v", written)
    _print_worst("app128-" + form, ft, rd)


@pytest.mark.parametrize("rd", [128, 64])
def test_rope_standalone_and_fused_agree(rd):
    """b2_rotary: Q and K heads within both bounds, V and dims >= rotary_dim bit-identical; followed by an append without
    rotary it writes the same bits as the fused append (q_out and the span rows)."""
    from b200spark import ops
    ft = torch.bfloat16
    B, slots_n = len(G.ROPE_POS), NH + 2 * NG
    pos = torch.tensor(G.ROPE_POS, dtype=torch.int32, device="cuda")
    for base in G.ROPE_BASES:
        x = _qkv(B, slots_n, 128, ft, seed=rd)
        xd = G.to_ft(x.reshape(B, -1), ft).cuda()
        r = ops.rotary(xd.clone(), pos, NH, NG, base=base, rotary_dim=rd)
        torch.cuda.synchronize()
        got = _np(r).reshape(B, slots_n, 128)
        _rope_check("b2_rotary", got[:, :NH + NG], x[:, :NH + NG], np.array(G.ROPE_POS), base, rd, ft)
        assert np.array_equal(got[:, NH + NG:], x[:, NH + NG:])
        slots = [[p] for p in G.ROPE_POS]
        plain, fused = _Pages(slots, NH, NG, 128, ft), _Pages(slots, NH, NG, 128, ft)
        q1 = ops.cache_append(plain, r, pos)
        q2 = ops.cache_append(fused, xd, pos, rope=(base, rd))
        torch.cuda.synchronize()
        assert torch.equal(q1.view(torch.int16), q2.view(torch.int16)), base
        for which in "kv":  # the same page layout: the pools must match byte for byte
            assert torch.equal(plain.pools[which].cpu(), fused.pools[which].cpu()), (base, which)
    _print_worst("b2_rotary", ft, rd)


@pytest.mark.parametrize("rd", [64, 32])
def test_rope_append_head64(rd):
    """The head-64 append (14 / 2 heads, bf16): the same bounds, V and the unrotated dims bit-identical, no other byte
    changes."""
    from b200spark import ops
    ft, nH, nG = torch.bfloat16, 14, 2
    B = len(G.ROPE_POS)
    old = torch.tensor(G.ROPE_POS, dtype=torch.int32, device="cuda")
    for base in G.ROPE_BASES:
        slots = [[p] for p in G.ROPE_POS]
        cache = _Pages(slots, nH, nG, 64, ft)
        x = _qkv(B, nH + 2 * nG, 64, ft, seed=64 + rd)
        qo = ops.cache_append(cache, G.to_ft(x.reshape(B, -1), ft).cuda(), old, rope=(base, rd))
        torch.cuda.synchronize()
        pos = np.array(G.ROPE_POS)
        _rope_check("app64", _np(qo).reshape(B, nH, 64), x[:, :nH], pos, base, rd, ft)
        k = np.concatenate([cache.rows("k", b, slots[b]) for b in range(B)])
        v = np.concatenate([cache.rows("v", b, slots[b]) for b in range(B)])
        _rope_check("app64", k, x[:, nH:nH + nG], pos, base, rd, ft)
        assert np.array_equal(v, x[:, nH + nG:])
        written = [(b, p) for b, p in enumerate(G.ROPE_POS)]
        assert cache.untouched("k", written) and cache.untouched("v", written)
    _print_worst("app64", ft, rd)


# ---------------------------------------------------------------- argmax
def _argmax_ft(logits, n, id_offset):
    """b2_argmax_ft with vals_out over the first n columns of logits (row stride logits.stride(0))"""
    from b200spark import _lib, ops
    B = logits.shape[0]
    ids = torch.full((B,), -1, dtype=torch.int64, device="cuda")
    vals = torch.zeros(B, dtype=torch.float32, device="cuda")
    _lib.check(_lib.lib.b2_argmax_ft(ops._ptr(ids), ops._ptr(vals), ops._ptr(logits), B, n, logits.stride(0), id_offset, ops._ft(logits),
                                     ops._stream()), "b2_argmax_ft")
    return ids.cpu().numpy(), vals.cpu().numpy()


def _same_vals(a, b):
    return np.array_equal(a, b, equal_nan=True)


@pytest.mark.parametrize("n", G.ARGMAX_N)
@pytest.mark.parametrize("dt", ["bf16", "fp16"])
def test_argmax(dt, n):
    """Every row kind (ties decided in one thread, across lanes, across warps and in the final warp reduction, first and
    last, a constant row, all -inf, +inf, all NaN, some NaN) at batch 1 / 64 / 65, ld = n + 5 with larger values, +inf and
    NaN planted in the padding, id_offset 0 and 1000003: ids and vals_out exact, every id in [id_offset, id_offset + n)."""
    from b200spark import ops
    ft = G.FTS[dt]
    x = G.argmax_batch(n, 65, 5, seed=n)
    lg = G.to_ft(x, ft).cuda()
    xr = _np(lg)
    for batch in G.ARGMAX_BATCH:
        view = lg[:batch, :n]
        assert view.stride(0) == n + 5
        want, wvals = G.argmax_ref(xr[:batch], n)
        assert np.array_equal(ops.argmax(view).cpu().numpy(), want), batch
        for off in (0, 1000003):
            ids, vals = _argmax_ft(view, n, off)
            assert np.array_equal(ids, want + off), (batch, off)
            assert _same_vals(vals, wvals), batch
            assert ((ids >= off) & (ids < off + n)).all()
    kinds = [G.ARGMAX_KINDS[r % len(G.ARGMAX_KINDS)] for r in range(65)]
    ids, _ = _argmax_ft(lg[:, :n], n, 7)
    assert all(ids[r] == 7 for r, k in enumerate(kinds) if k in ("nan_all", "neg_inf", "equal"))  # their first index


@pytest.mark.parametrize("tp", [2, 4, 8])
@pytest.mark.parametrize("n", [128256, 151936, 152064])
def test_argmax_shard_merge(n, tp):
    """Vocab split over tp shards: argmax_shard of each shard (a strided view of the whole row, id_offset = the shard
    start), the pairs stacked as after the all-gather, argmax_merge == argmax of the whole row.  Winners on shard edges,
    ties across shards and NaN in two shards resolve to the lowest rank."""
    from b200spark import ops
    rng = np.random.default_rng(n + tp)
    x = np.stack([G.tp_row(k, n, tp, rng) for k in G.TP_KINDS])
    lg = G.to_ft(x, torch.bfloat16).cuda()
    xr = _np(lg)
    B = len(G.TP_KINDS)
    bounds = G.shard_bounds(n, tp)
    all_ids = torch.empty(tp, B, dtype=torch.int64, device="cuda")
    all_vals = torch.empty(tp, B, dtype=torch.float32, device="cuda")
    for r, (s, e) in enumerate(bounds):
        ops.argmax_shard(lg[:, s:e], s, all_ids[r], all_vals[r])
    merged = ops.argmax_merge(all_vals, all_ids, torch.empty(B, dtype=torch.int64, device="cuda"))
    whole = ops.argmax(lg)
    torch.cuda.synchronize()
    for r, (s, e) in enumerate(bounds):
        want, wv = G.argmax_ref(xr[:, s:e], e - s, s)
        assert np.array_equal(all_ids[r].cpu().numpy(), want), r
        assert _same_vals(all_vals[r].cpu().numpy(), wv), r
    want, _ = G.argmax_ref(xr, n)
    assert np.array_equal(merged.cpu().numpy(), want), dict(zip(G.TP_KINDS, merged.cpu().tolist()))
    assert np.array_equal(whole.cpu().numpy(), want)


# ---------------------------------------------------------------- binary, embedding, lens_add
@pytest.mark.parametrize("n", G.BINARY_N)
@pytest.mark.parametrize("dt", ["bf16", "fp16"])
def test_binary(dt, n):
    """ADD and MUL bit-exact against the fp32 op rounded once, including out == a and out == b, and (fp16) overflow to +-inf"""
    from b200spark import BIN_ADD, BIN_MUL, ops
    ft = G.FTS[dt]
    rng = np.random.default_rng(n)
    a, b = rng.standard_normal(n) * 4, rng.standard_normal(n) * 4
    if dt == "fp16":
        k = rng.choice(n, min(3, n), replace=False)
        a[k], b[k] = [60000.0, -60000.0, 300.0][:len(k)], [60000.0, -60000.0, -300.0][:len(k)]
    at, bt = G.to_ft(a, ft), G.to_ft(b, ft)
    ad, bd = at.cuda(), bt.cuda()
    for op in (BIN_ADD, BIN_MUL):
        want = G.binary_ref(at, bt, op == BIN_ADD, ft).view(torch.int16)
        assert torch.equal(ops.binary(ad, bd, op).cpu().view(torch.int16), want), op
        o = ad.clone()
        assert torch.equal(ops.binary(o, bd, op, out=o).cpu().view(torch.int16), want), op
        o = bd.clone()
        assert torch.equal(ops.binary(ad, o, op, out=o).cpu().view(torch.int16), want), op
    if dt == "fp16" and n >= 3:
        s = ops.binary(ad, bd, BIN_ADD).cpu()
        assert torch.isinf(s).sum() >= 2


@pytest.mark.parametrize("hidden", G.EMBED_HIDDEN)
@pytest.mark.parametrize("dt", ["bf16", "fp16"])
def test_embedding(dt, hidden):
    """rows 0 and vocab - 1, repeated ids: the table's bits"""
    from b200spark import ops
    ft = G.FTS[dt]
    vocab = 152064 if hidden == 8 else 3001
    g = torch.Generator().manual_seed(hidden)
    table = torch.randn(vocab, hidden, generator=g).to(ft)
    ids = torch.tensor([0, vocab - 1, 5, 5, vocab - 1, 0] + torch.randint(0, vocab, (7,), generator=g).tolist(), dtype=torch.int64)
    out = ops.embedding(table.cuda(), ids.cuda())
    assert out.dtype == ft and torch.equal(out.cpu().view(torch.int16), table[ids].view(torch.int16))


def test_lens_add():
    from b200spark import ops
    lens = torch.randint(100, 100000, (129,), dtype=torch.int32, generator=torch.Generator().manual_seed(1))
    d = lens.cuda()
    ops.lens_add(d, -3)
    assert torch.equal(d.cpu(), lens - 3)
    ops.lens_add(d, 7)
    assert torch.equal(d.cpu(), lens + 4)
