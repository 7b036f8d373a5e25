"""GPU: SpanAttention with needle inputs (tests/attn_needles.py) at every tile, span and split-KV piece edge.

One token per needle carries O(1) of its head's softmax weight, so a token dropped, counted twice or read one position
off moves the output by >= 20 envelopes (checked on every launch, on the device's own cache bytes).  The oracle is fp64
attention over those bytes; the bound per element is the attention contract (2e-3 + 2^-7 |ref| in bf16, 2^-9 in fp16) plus
the rounding of the probabilities the P V MMA multiplies (attn_needles.evaluate).  Every launch runs twice and must repeat
bit for bit.  Head-128 caches are written with the prefill writer (bit-identical to appends: test_ref_pin_gpu.py,
test_kv_fp8_gpu.py); head-64 spans are written into the span pages directly (there is no head-64 prefill writer)."""
import math

import numpy as np
import pytest
import torch

import attn_needles as A

pytestmark = pytest.mark.gpu


def _grid(attn, B, max_len, hpg):
    """CTAs of the handle's launch: its workspace holds two level-0 and two level-1 partials of hpg x (128 + 2) fp32 per
    CTA, plus 256 bytes of alignment slack"""
    per = 2 * 2 * hpg * (128 + 2) * 4
    ws = attn.workspace_bytes(B, max_len) - 256
    assert ws > 0 and ws % per == 0, ws
    return ws // per


def _spans(pool, perm, cache, b, W):
    return [pool[int(perm[b, si]) * cache.stride:int(perm[b, si]) * cache.stride + cache.span_bytes]
            for si in range((W + cache.cfg.span_len - 1) // cache.cfg.span_len)]


def _write(cache, case, which, rows):
    """rows: per sequence [W_b, nG, head] fp32 values of the model type"""
    from b200spark import ops
    if case.head == 128:
        for b, x in enumerate(rows):
            ops.context_copy(cache, which, b, torch.from_numpy(x.reshape(x.shape[0], -1)).to(case.dtype).cuda())
        return
    pool_t, perm = (cache.k_pool, cache.perm_k) if which == "k" else (cache.v_pool, cache.perm_v)
    pool = pool_t.cpu().numpy()
    span, nG = case.span, case.nG
    for b, x in enumerate(rows):
        bits = torch.from_numpy(np.ascontiguousarray(x)).to(torch.bfloat16).view(torch.int16).numpy().view(np.uint16)
        for si, buf in enumerate(_spans(pool, perm, cache, b, x.shape[0])):
            n = min(span, x.shape[0] - si * span)
            buf.view(np.uint16).reshape(nG, span, case.head)[:, :n] = bits[si * span:si * span + n].transpose(1, 0, 2)
    pool_t.copy_(torch.from_numpy(pool))


def _run(case, monkeypatch, expect_grid=None):
    from b200spark import ops
    if case.max_pieces:
        monkeypatch.setenv("B2_ATTN_MAX_PIECES", str(case.max_pieces))
    if case.ctas_per_sm:
        monkeypatch.setenv("B2_ATTN_CTAS_PER_SM", str(case.ctas_per_sm))
    prob = case.problem()
    B, W = len(case.lens), prob.written
    max_len = max(W)
    cache = ops.SpanCache(B, max_len, case.nH, case.nG, case.span, case.mode, fill=case.fill, dtype=case.dtype, head=case.head)
    attn = ops.SpanAttn(cache.cfg, B)  # created after the knobs are set: they are read when the handle is made
    ws = ops.Workspace()
    grid = _grid(attn, B, max_len, case.hpg)
    if expect_grid is not None:
        assert grid == expect_grid, (grid, expect_grid)
    lens_d = torch.tensor(case.lens, dtype=torch.int32, device="cuda")
    worst, least_teeth, rounds = 0.0, math.inf, case.rounds(grid)
    for needles, stale in rounds:
        k_rows, v_rows, q = prob.rows(needles)
        _write(cache, case, "k", k_rows)
        _write(cache, case, "v", v_rows)
        qd = torch.from_numpy(q.reshape(B, -1)).to(case.dtype).cuda()
        out = attn(qd, cache, lens_d, max_len, ws)
        out2 = attn(qd, cache, lens_d, max_len, ws)
        torch.cuda.synchronize()
        assert out.dtype == case.dtype and torch.equal(out, out2), case.name  # deterministic, counters re-armed
        got = out.float().cpu().numpy().reshape(B, case.nH, case.head).astype(np.float64)
        kp, vp = cache.k_pool.cpu().numpy(), cache.v_pool.cpu().numpy()
        kc, ks, vc, vs = [], [], [], []
        for b in range(B):
            c, s = A.from_spans(_spans(kp, cache.perm_k, cache, b, W[b]), case.mode, case.span, case.nG, W[b], case.head, case.dtype)
            kc.append(c); ks.append(s)
            c, s = A.from_spans(_spans(vp, cache.perm_v, cache, b, W[b]), case.mode, case.span, case.nG, W[b], case.head, case.dtype)
            vc.append(c); vs.append(s)
        res = A.evaluate(prob, q, kc, ks, vc, vs, case.mode, needles, stale=stale)
        # the read-back cache keeps its sensitivity: every needle still has teeth, honest rounding fits the envelope
        if max(case.lens) > 1:
            assert res.teeth >= A.TEETH, (case.name, res.teeth, res.weakest)
        assert res.honest <= 1.0, (case.name, res.honest)
        assert np.isfinite(got).all(), case.name
        ratio = np.abs(got - res.ref) / res.env
        least_teeth = min(least_teeth, res.teeth)
        if ratio.max() > worst:
            worst = float(ratio.max())
        b, h, d = np.unravel_index(int(np.argmax(ratio)), ratio.shape)
        assert ratio.max() <= 1.0, (case.name, "seq %d head %d dim %d" % (b, h, d), float(got[b, h, d]), float(res.ref[b, h, d]),
                                    [n for n in needles if n[:2] == (b, h)])
    print("%-28s grid %4d  %3d launches  worst error/envelope %.3f  least teeth %.0f" % (case.name, grid, len(rounds), worst, least_teeth))


@pytest.mark.parametrize("case", A.tile_cases(), ids=lambda c: c.name)
def test_needles_every_tile_and_span_edge(case, monkeypatch):
    """Default knobs: needles on 0, len - 1 and the first and last token of every tile and every span.  Piece edges are
    tile edges, so whatever the grid, every piece edge carries a needle."""
    _run(case, monkeypatch)


@pytest.mark.parametrize("mode", [A.NONE, A.I8, A.FP8])
def test_needles_merge_shapes(mode, monkeypatch):
    """B2_ATTN_CTAS_PER_SM=1 (grid = the SM count): the mirror must find every merge shape in these launches before they
    run (1 piece inside a CTA shared by several (sequence, kv-head)s, 2 pieces starting mid-CTA, 16 and 17 pieces, 8q and
    8q+1 pieces with the next (sequence, kv-head) starting in the last CTA, Tc = 1 with > 100 pieces)."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    found = set()
    for lens, nH, nG, mp in A.merge_shape_cases(sms):
        dec = A.decompose(lens, nG, sms, mp)
        A.check_decomposition(dec, lens)
        found |= A.shapes(dec)
    assert found == A.MERGE_SHAPES, A.MERGE_SHAPES - found
    for case in A.merge_cases(sms, mode):
        with monkeypatch.context() as m:
            _run(case, m, expect_grid=sms)


@pytest.mark.parametrize("case", A.long_cases(), ids=lambda c: c.name)
def test_needles_ctx_32768(case, monkeypatch):
    _run(case, monkeypatch)


@pytest.mark.parametrize("case", A.stale_cases(), ids=lambda c: c.name)
def test_needles_stale_rows(case, monkeypatch):
    """300 tokens written, attention over 100 / 128: needles at token L1 and in a later span must not count; the result is
    attention over [0, L1).  Finite stale data (the 0xFF NaN pool is test_attn_gpu's)."""
    _run(case, monkeypatch)


@pytest.mark.parametrize("case", A.head64_cases(), ids=lambda c: c.name)
def test_needles_head64(case, monkeypatch):
    """Head 64 (one CTA per (sequence, kv-head), 32 tokens per step): needles at 31 / 32, every span edge, 0 and len - 1,
    over a 0xFF-filled pool."""
    _run(case, monkeypatch)


def _bf16(x):
    return torch.from_numpy(np.ascontiguousarray(x, np.float32)).to(torch.bfloat16).float().numpy()


def _bf16_ulp(v):
    return 2.0 ** (np.floor(np.log2(np.maximum(np.abs(v), 2.0 ** -126))) - 7)


@pytest.mark.parametrize("rotary_dim", [None, 64, 32])
def test_head64_append(rotary_dim):
    """cache_append at head 64 (Qwen2-0.5B: 14 / 2 heads, span 16) at positions 0, 15, 16 (a span edge) and 30000 into a
    0xFF pool.  Without rotary, q_out and the span rows are the input bits.  With rotary over 64 or 32 dims: within 1 bf16
    ulp of the kernel's fp32 formula (inv = exp2(-log2(base) * 2i / rotary_dim), angle = fl32(pos * inv), rounded once),
    widened at large positions by what exp2f's 2-ulp error moves the angle; within 2e-2 of fp64 NeoX (the bound of the
    head-128 rotary test); dims beyond rotary_dim and the V rows bit-identical to the input; no other span row touched."""
    from b200spark import ops
    nH, nG, span, head, base = 14, 2, 16, 64, 1e6
    pos = np.array([0, 15, 16, 30000])
    B = len(pos)
    cache = ops.SpanCache(B, 30016, nH, nG, span, A.NONE, fill=0xFF, head=head)
    rng = np.random.default_rng(64 + (rotary_dim or 0))
    x = _bf16(rng.standard_normal((B, nH + 2 * nG, head)) * 2)
    qo = ops.cache_append(cache, torch.from_numpy(x.reshape(B, -1)).to(torch.bfloat16).cuda(),
                          torch.tensor(pos, dtype=torch.int32, device="cuda"), rope=(base, rotary_dim) if rotary_dim else None)
    torch.cuda.synchronize()
    qk = x[:, :nH + nG]
    want, tol, want64 = qk.copy(), np.zeros_like(qk), qk.astype(np.float64).copy()
    if rotary_dim:
        half = rotary_dim // 2
        i = np.arange(rotary_dim) % half
        inv = np.exp2(-np.log2(np.float32(base)) * (np.float32(2.0) * i.astype(np.float32) / np.float32(rotary_dim))).astype(np.float32)
        ang = (pos.astype(np.float32)[:, None] * inv[None]).astype(np.float32)          # [B, rotary_dim]
        cs, sn = np.cos(ang.astype(np.float64))[:, None], np.sin(ang.astype(np.float64))[:, None]
        a, o = qk[..., :rotary_dim], np.concatenate([-qk[..., half:rotary_dim], qk[..., :half]], -1)
        want[..., :rotary_dim] = _bf16((a * cs + o * sn).astype(np.float32))
        dang = pos[:, None, None] * inv[None, None].astype(np.float64) * 2.0 ** -22    # 2 ulp of exp2f in the angle
        tol[..., :rotary_dim] = _bf16_ulp(want[..., :rotary_dim]) + (np.abs(a) + np.abs(o)) * dang
        inv64 = base ** (-np.arange(half, dtype=np.float64) * 2 / rotary_dim)
        ang64 = pos[:, None].astype(np.float64) * np.concatenate([inv64, inv64])[None]
        a64, o64 = want64[..., :rotary_dim].copy(), np.concatenate([-want64[..., half:rotary_dim], want64[..., :half]], -1)
        want64[..., :rotary_dim] = a64 * np.cos(ang64)[:, None] + o64 * np.sin(ang64)[:, None]
    got_q = qo.float().cpu().numpy().reshape(B, nH, head)
    assert np.all(np.abs(got_q - want[:, :nH]) <= tol[:, :nH])
    assert np.abs(got_q - want64[:, :nH]).max() <= 2e-2
    if rotary_dim:
        assert np.array_equal(got_q[..., rotary_dim:], x[:, :nH, rotary_dim:])
    else:
        assert np.array_equal(got_q, x[:, :nH])
    for b, p in enumerate(pos):
        si, r = p // span, p % span
        for which, rows, t in (("k", want[b, nH:], tol[b, nH:]), ("v", x[b, nH + nG:], 0.0)):
            raw = cache.span_view(which, b, si).cpu().view(torch.bfloat16).reshape(nG, span, head)
            got = raw[:, r].float().numpy()
            assert np.all(np.abs(got - rows) <= t), (which, p)
            if which == "v" or not rotary_dim:
                assert np.array_equal(got, rows), (which, p)
            else:
                assert np.array_equal(got[:, rotary_dim:], rows[:, rotary_dim:]), (which, p)
                assert np.abs(got - want64[b, nH:]).max() <= 2e-2
            others = np.delete(raw.view(torch.int16).numpy(), r, axis=1)
            assert (others == -1).all(), (which, p)  # every other row still 0xFFFF
