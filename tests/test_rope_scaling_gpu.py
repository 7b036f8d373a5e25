"""GPU: the scaled rotary from a caller-given frequency table (b2_rope_table).  The table form of the span-cache append
against the restatement's bound (tests/rope_scaling_ref.py) and against b2_rotary_table followed by the append without
rotary, bit for bit, over every step form, KV mode, FT, Q/K norm and rotary width, with shared and per-sequence tables;
b2_rotary_table at positions up to 200000; guard frames, repeat runs and CUDA-graph replay; the base-frequency table
against the computed base frequencies."""
import ctypes as C

import numpy as np
import pytest
import torch

import glue_ref as G
import rope_scaling_ref as R

pytestmark = pytest.mark.gpu

NH, NG, SPAN = 4, 2, 16
SLOTS = NH + 2 * NG
FORMS = {"single": (1, None), "chain": (3, None), "tree": (4, [0, 0, 0, 1])}  # q_len, parents (depths 0, 1, 1, 2)
MODES = ["none", "i8", "u4", "fp8"]
EPS = 1e-6


def _np(t):
    return t.float().cpu().numpy().astype(np.float64)


class _Pages:
    """Span tables for appends at far positions without a whole cache (as test_glue_gpu's): each span a row lands in gets
    its own page, every other table entry points at one shared guard page; every page starts 0xFF."""

    def __init__(self, slots, mode, dt):
        from b200spark import _lib
        qm = {"none": _lib.KV_NONE, "i8": _lib.KV_I8, "u4": _lib.KV_U4, "fp8": _lib.KV_FP8}[mode]
        max_spans = max(max(s) for s in slots) // SPAN + 1
        self.cfg = _lib.SpanCfg({torch.bfloat16: _lib.DT_BF16, torch.float16: _lib.DT_F16}[dt], qm, NH, NG, 128, SPAN, max_spans, 0)
        self.span_bytes = _lib.lib.b2_span_bytes(C.byref(self.cfg))
        self.stride = (self.span_bytes + 255) // 256 * 256
        self.dt, self.page = dt, {}
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
        """[len(slots), nG, 128] values of the given slots of sequence b (16-bit spans only)"""
        pool = self.pools[which].cpu()
        out = []
        for s in slots:
            off = self.page[(b, s // SPAN)] * self.stride
            out.append(pool[off:off + self.span_bytes].view(self.dt).reshape(NG, SPAN, 128)[:, s % SPAN].float().numpy())
        return np.stack(out)


def _tables(B, rd, per_seq, device="cuda"):
    """(inv [rd/2] or [B, rd/2] viewed out of [B, rd/2 + 4] (a row stride above rd/2), attn_factor, host rows [S, rd/2]): a
    shared Qwen2.5 table, or YaRN factors 2, 3, 4, ... per sequence"""
    from b200spark import ops
    if not per_seq:
        inv, af = ops.rope_table(R.QWEN25[1], 1e6, rd)
        return inv.to(device), af, inv.numpy()[None]
    rows = [ops.rope_table(dict(R.QWEN25[1], factor=2.0 + b % 5), 1e6, rd)[0] for b in range(B)]
    pad = torch.full((B, rd // 2 + 4), float("nan"))
    pad[:, :rd // 2] = torch.stack(rows)
    return pad.to(device)[:, :rd // 2], ops.rope_table(R.QWEN25[1], 1e6, rd)[1], torch.stack(rows).numpy()


def _step(form, ft, rd, seed, pos0=G.ROPE_POS):
    q_len, parents = FORMS[form]
    B = len(pos0)
    depth = [0] * q_len
    for t in range(1, q_len):
        depth[t] = depth[parents[t]] + 1 if parents else t
    rng = np.random.default_rng(seed)
    x = G.ft_values(rng.standard_normal((B * q_len, SLOTS, 128)) * 2, ft)
    kw = {} if q_len == 1 else {"q_len": q_len}
    if parents:
        kw["parents"] = torch.tensor([parents] * B, dtype=torch.int32, device="cuda")
    slots = [[p + t for t in range(q_len)] for p in pos0]
    rpos = np.array([p + depth[t] for p in pos0 for t in range(q_len)])
    seq = np.repeat(np.arange(B), q_len)
    return x, kw, slots, rpos, seq


def _guarded_q(rows, ft):
    """q_out inside a frame of guard rows (value -7)"""
    buf = torch.full((rows + 2, NH * 128), -7.0, dtype=ft, device="cuda")
    return buf, buf[1:-1]


def _fused_and_composed(form, mode, ft, rd, per_seq, qkn, seed):
    from b200spark import ops
    x, kw, slots, rpos, seq = _step(form, ft, rd, seed)
    B, rows = len(slots), x.shape[0]
    xd = G.to_ft(x.reshape(rows, -1), ft).cuda()
    old = torch.tensor(G.ROPE_POS, dtype=torch.int32, device="cuda")
    inv, af, host = _tables(B, rd, per_seq)
    g = torch.Generator(device="cuda").manual_seed(seed)
    norm = None
    if qkn:
        norm = tuple((1 + 0.1 * torch.randn(128, generator=g, device="cuda")).to(ft) for _ in range(2)) + (EPS,)
    fused, buf = _Pages(slots, mode, ft), _guarded_q(rows, ft)
    ops._cache_append(fused, xd, old, q_out=buf[1], rope=(inv, af), qk_norm=norm, **kw)
    # composed: [norm] -> b2_rotary_table (the sequence's table row for every one of its tokens) -> append without rotary
    y = ops.qk_rmsnorm(xd, NH, NG, norm[0], norm[1], EPS) if qkn else xd.clone()
    tab = inv if not per_seq else inv.repeat_interleave(rows // B, 0)
    ops.rotary(y, torch.tensor(rpos, dtype=torch.int32, device="cuda"), NH, NG, table=(tab, af))
    comp = _Pages(slots, mode, ft)
    qc = ops._cache_append(comp, y, old, **kw)
    torch.cuda.synchronize()
    return dict(x=x, y=y, slots=slots, rpos=rpos, seq=seq, host=host, af=af, fused=fused, buf=buf, comp=comp, qc=qc)


@pytest.mark.parametrize("rd", [128, 64])
@pytest.mark.parametrize("qkn", [False, True])
@pytest.mark.parametrize("dt", ["bf16", "fp16"])
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("form", list(FORMS))
def test_table_append(form, mode, dt, qkn, rd):
    """fused = composed bit for bit (span bytes, {zero, scale}, q_out); the guard rows around q_out untouched; without the
    norm, q_out (and the K rows of 16-bit spans) within the restatement's bound, V rows as given"""
    ft = G.FTS[dt]
    for per_seq in (False, True):
        r = _fused_and_composed(form, mode, ft, rd, per_seq, qkn, seed=len(form) * 7 + rd + per_seq)
        buf, q = r["buf"]
        assert torch.equal(buf[0], torch.full_like(buf[0], -7.0)) and torch.equal(buf[-1], torch.full_like(buf[-1], -7.0))
        assert torch.equal(q.view(torch.int16), r["qc"].view(torch.int16)), per_seq
        for w in "kv":
            assert torch.equal(r["fused"].pools[w], r["comp"].pools[w]), (per_seq, w)
        if qkn:
            continue  # the rotary of a normalised row: the composed path's b2_rotary_table, bounded where qkn is off
        xin = r["x"]
        Y, D = R.table_formula(xin[:, :NH + NG], r["rpos"], r["host"], r["af"], NH, rd, seq=r["seq"])
        assert R.ratio(_np(q).reshape(-1, NH, 128), Y[:, :NH], D[:, :NH], ft).max() <= 1.0, per_seq
        if mode == "none":
            B = len(r["slots"])
            k = np.concatenate([r["fused"].rows("k", b, r["slots"][b]) for b in range(B)])
            v = np.concatenate([r["fused"].rows("v", b, r["slots"][b]) for b in range(B)])
            assert R.ratio(k, Y[:, NH:], D[:, NH:], ft).max() <= 1.0, per_seq
            assert np.array_equal(v, r["x"][:, NH + NG:])


@pytest.mark.parametrize("rd", [128, 64])
@pytest.mark.parametrize("dt", ["bf16", "fp16"])
def test_rotary_table_far_positions(dt, rd):
    """b2_rotary_table up to position 200000, shared and per-row tables: q and k heads within the bound, V heads and the
    dims >= rotary_dim keep their bits"""
    from b200spark import ops
    ft = G.FTS[dt]
    pos = G.ROPE_POS + [200000]
    rng = np.random.default_rng(rd)
    x = G.ft_values(rng.standard_normal((len(pos), SLOTS, 128)) * 2, ft)
    for per_seq in (False, True):
        inv, af, host = _tables(len(pos), rd, per_seq)
        y = ops.rotary(G.to_ft(x.reshape(len(pos), -1), ft).cuda(), torch.tensor(pos, dtype=torch.int32, device="cuda"), NH, NG,
                       table=(inv, af))
        torch.cuda.synchronize()
        got = _np(y).reshape(len(pos), SLOTS, 128)
        Y, D = R.table_formula(x[:, :NH + NG], np.array(pos), host, af, NH, rd, seq=np.arange(len(pos)))
        assert R.ratio(got[:, :NH + NG], Y, D, ft).max() <= 1.0, per_seq
        assert np.array_equal(got[:, NH + NG:], x[:, NH + NG:])
        assert np.array_equal(got[..., rd:], x[..., rd:])


@pytest.mark.parametrize("form", list(FORMS))
def test_repeat_and_graph_replay(form):
    """the same inputs give the same bytes on a second run and from a captured CUDA graph"""
    from b200spark import ops
    ft = torch.bfloat16
    x, kw, slots, rpos, seq = _step(form, ft, 128, seed=5)
    rows = x.shape[0]
    xd = G.to_ft(x.reshape(rows, -1), ft).cuda()
    old = torch.tensor(G.ROPE_POS, dtype=torch.int32, device="cuda")
    inv, af, _ = _tables(len(slots), 128, True)
    runs = []
    for graph in (False, False, True):
        c = _Pages(slots, "i8", ft)
        q = torch.empty(rows, NH * 128, dtype=ft, device="cuda")
        if not graph:
            ops._cache_append(c, xd, old, q_out=q, rope=(inv, af), **kw)
        else:
            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                gr = torch.cuda.CUDAGraph()
                with torch.cuda.graph(gr, stream=s):
                    ops._cache_append(c, xd, old, q_out=q, rope=(inv, af), **kw)
            torch.cuda.synchronize()
            gr.replay()
        torch.cuda.synchronize()
        runs.append((q.clone(), c.pools["k"].clone(), c.pools["v"].clone()))
    for r in runs[1:]:
        assert all(torch.equal(a, b) for a, b in zip(runs[0], r))


@pytest.mark.parametrize("rd", [128, 64])
def test_base_table_agrees_with_base_path(rd):
    """the table of the unscaled frequencies (host fp64, rounded once) and the computed ones (device exp2f) at positions
    below the native context: both within the fp64 NeoX bound, and apart by at most the sum of their allowances"""
    from b200spark import ops
    ft, base = torch.bfloat16, 1e6
    pos = [p for p in G.ROPE_POS if p < 32768]
    slots = [[p] for p in pos]
    x = G.ft_values(np.random.default_rng(rd).standard_normal((len(pos), SLOTS, 128)) * 2, ft)
    xd = G.to_ft(x.reshape(len(pos), -1), ft).cuda()
    old = torch.tensor(pos, dtype=torch.int32, device="cuda")
    inv, af = ops.rope_table(None, base, rd, device="cuda")
    a, b = _Pages(slots, "none", ft), _Pages(slots, "none", ft)
    qa = ops._cache_append(a, xd, old, rope=(inv, af))
    qb = ops._cache_append(b, xd, old, rope=(base, rd))
    torch.cuda.synchronize()
    Y, D = G.rope_neox64(x[:, :NH], np.array(pos)[:, None], base, rd)
    ya, yb = _np(qa).reshape(-1, NH, 128), _np(qb).reshape(-1, NH, 128)
    allow = G.ulp(np.abs(Y) + D, ft) / 2 + D
    assert G.rope_ratio(ya, Y, D, ft).max() <= 1.0 and G.rope_ratio(yb, Y, D, ft).max() <= 1.0
    assert np.all(np.abs(ya - yb) <= 2 * allow)
    print("base table vs computed base frequencies: %d of %d q values differ" % (int((ya != yb).sum()), ya.size))
