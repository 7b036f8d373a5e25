"""GPU: multi-token decode steps (speculative decoding) — span append of q_len tokens per sequence, attention with a
per-row causal limit, greedy acceptance on the device, and the decode stack's verify step.

Attention is checked against fp64 attention (tests/spec_ref.py) over the cache bytes read back from the device, with the
bound of test_attn_gpu.py's quantized tests: 2e-3 + 2^-7 |ref| (bf16 output; fp16 output 2^-9).  Rows that see at most one
tile (64 tokens) add the rounding of the probabilities the P V MMA multiplies, u_P sum_j p_j |V_j| (u_P as in
tests/attn_needles.py): there a single probability carries O(1) weight.  The causal limit itself is checked with needles
(tests/attn_needles.py), which a limit off by one token moves by >= 20 envelopes at any length."""
import math
import types

import numpy as np
import pytest
import torch

import attn_needles as A
import spec_ref as S
from oracle import kvcache_ref as KV

pytestmark = pytest.mark.gpu

MODES = [KV.QUANT_NONE, KV.QUANT_I8, KV.QUANT_U4, 3]  # 3: fp8 e4m3


def _rand(rng, shape, dtype):
    return torch.from_numpy(rng.standard_normal(shape).astype(np.float32)).to(dtype).cuda()


def _filled_cache(mode, lens, nH, nG, span, dtype, seed, max_len):
    """Spans written by the prefill writer with N(0,1) rows, plus oracle caches holding the device's own span bytes."""
    from b200spark import ops
    rng = np.random.default_rng(seed)
    B = len(lens)
    cache = ops.SpanCache(B, max_len, nH, nG, span, mode, fill=0xFF, dtype=dtype)
    for b, L in enumerate(lens):
        ops.context_copy(cache, "k", b, _rand(rng, (L, nG * 128), dtype))
        ops.context_copy(cache, "v", b, _rand(rng, (L, nG * 128), dtype))
    torch.cuda.synchronize()
    refs = []
    for which in ("k", "v"):
        ref = KV.SpanCacheRef(mode if mode != 3 else KV.QUANT_I8, span, nG, ft="fp16" if dtype == torch.float16 else "bf16")
        for b, L in enumerate(lens):
            ref.add_sequence()
            ref.spans[b] = [cache.span_view(which, b, si).cpu().numpy().copy() for si in range(-(-L // span))]
        refs.append(ref)
    return cache, refs[0], refs[1]


def _dense_fp8(ref):
    """fp8 spans share the I8 layout: decode the e4m3 codes times the scale (zero = 0)"""
    def dense(b, length, ref=ref):
        S_, G = ref.span_len, ref.n_groups
        out = np.zeros((G, length, 128), np.float32)
        for si in range(-(-length // S_)):
            buf = ref.spans[b][si]
            n = min(S_, length - si * S_)
            codes = torch.from_numpy(buf[:S_ * G * 128].copy()).view(torch.float8_e4m3fn).float().numpy().reshape(G, S_, 128)
            prm = buf[S_ * G * 128:].view(np.float32).reshape(G, S_, 2)
            out[:, si * S_: si * S_ + n] = codes[:, :n] * prm[:, :n, 1:2]
        return out
    ref.dense = dense
    return ref


def _check(got, ref, ref_abs, lens, T, mode, dtype):
    """got / ref / ref_abs [B, T, nH, 128]"""
    err = np.abs(got - ref)
    bound = 2e-3 + (2.0 ** -9 if dtype == torch.float16 else 2.0 ** -7) * np.abs(ref)
    u_p, _ = A.p_type(mode if mode != 3 else A.FP8, dtype, 128)
    lim = np.array([[S.row_limit(L, T, t) for t in range(T)] for L in lens])
    bound = bound + np.where(lim <= A.TILE, u_p, 0.0)[:, :, None, None] * ref_abs
    assert np.all(np.isfinite(got))
    worst = np.unravel_index(int(np.argmax(err - bound)), err.shape)
    assert np.all(err <= bound), ("seq %d token %d (limit %d) head %d dim %d" % (worst[0], worst[1], lim[worst[:2]], worst[2], worst[3]),
                                  float(err[worst]), float(bound[worst]))


# ---------------------------------------------------------------------------------------------------------------- append
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("span", [16, 128])
@pytest.mark.parametrize("rope", [False, True])
def test_append_tokens_equals_single_appends(mode, dtype, span, rope):
    """q_len rows per sequence in one call write the same span bytes, {zero, scale} and q rows as q_len single appends."""
    from b200spark import ops
    rng = np.random.default_rng(span + mode + (7 if rope else 0))
    nH, nG, T = 8, 2, 5
    old = [0, 13, span - 2, 2 * span - 1]  # ragged, crossing span boundaries
    B = len(old)
    a = ops.SpanCache(B, 3 * span, nH, nG, span, mode, fill=0xFF, dtype=dtype)
    s = ops.SpanCache(B, 3 * span, nH, nG, span, mode, fill=0xFF, dtype=dtype)
    qkv = _rand(rng, (B * T, (nH + 2 * nG) * 128), dtype)
    r = (1e6, 128) if rope else None
    old_d = torch.tensor(old, dtype=torch.int32, device="cuda")
    q_multi = ops.cache_append_tokens(a, qkv, old_d, T, rope=r)
    q_single = torch.empty_like(q_multi)
    rows = qkv.view(B, T, -1)
    for t in range(T):
        q1 = ops.cache_append(s, rows[:, t].contiguous(), old_d + t, rope=r)
        q_single.view(B, T, -1)[:, t] = q1
    torch.cuda.synchronize()
    assert torch.equal(a.k_pool, s.k_pool) and torch.equal(a.v_pool, s.v_pool)
    assert torch.equal(q_multi.view(torch.int16), q_single.view(torch.int16))


# ------------------------------------------------------------------------------------------------------------- attention
def _attn_case(mode, T, nH, nG, lens, span=16, dtype=torch.bfloat16, seed=0, max_pieces=None, monkeypatch=None):
    from b200spark import ops
    max_len = max(lens) + 1
    cache, kref, vref = _filled_cache(mode, lens, nH, nG, span, dtype, seed, max_len)
    if mode == 3:
        _dense_fp8(kref), _dense_fp8(vref)
    if max_pieces is not None:
        monkeypatch.setenv("B2_ATTN_MAX_PIECES", str(max_pieces))
    attn = ops.SpanAttn(cache.cfg, len(lens) * T)
    rng = np.random.default_rng(seed + 1)
    q = _rand(rng, (len(lens) * T, nH * 128), dtype)
    new_lens = torch.tensor(lens, dtype=torch.int32, device="cuda")
    ws = ops.Workspace()
    out = attn.run_tokens(q, cache, new_lens, T, max_len, ws)
    out2 = attn.run_tokens(q, cache, new_lens, T, max_len, ws)
    torch.cuda.synchronize()
    assert torch.equal(out, out2), "deterministic, counters re-armed"
    ref, ref_abs = S.attention_tokens(q.float().cpu().numpy().reshape(len(lens), T, nH, 128), kref, vref, lens, T, nH,
                                      1 / np.sqrt(128), with_abs=True)
    _check(out.float().cpu().numpy().reshape(len(lens), T, nH, 128), ref, ref_abs, lens, T, mode, dtype)
    return attn, cache, q, new_lens, out


@pytest.mark.parametrize("T", [1, 2, 3, 4, 8, 16])
@pytest.mark.parametrize("nH,nG", [(8, 8), (16, 4), (28, 4), (16, 2), (16, 1)])  # hpg 1, 4, 7, 8, 16
def test_attention_tokens_bf16(T, nH, nG):
    _attn_case(KV.QUANT_NONE, T, nH, nG, [T, T + 61, 64 + T, 200, 2049], seed=T * 31 + nH)


@pytest.mark.parametrize("mode", MODES[1:])
@pytest.mark.parametrize("T", [1, 4, 8])
@pytest.mark.parametrize("nH,nG", [(28, 4), (16, 1), (8, 8)])
def test_attention_tokens_quantized(mode, T, nH, nG):
    _attn_case(mode, T, nH, nG, [T, 65, 130, 2049], seed=T + nH + 5 * mode)


@pytest.mark.parametrize("mode", MODES)
def test_attention_tokens_fp16(mode):
    _attn_case(mode, 4, 28, 4, [4, 100, 700], dtype=torch.float16, seed=40 + mode)


@pytest.mark.parametrize("mode", [KV.QUANT_NONE, KV.QUANT_I8])
@pytest.mark.parametrize("cap", [4, 17])
def test_attention_tokens_piece_caps(mode, cap, monkeypatch):
    """B2_ATTN_MAX_PIECES forcing the direct (<= 16 pieces) and the two-level merge"""
    _attn_case(mode, 4, 28, 4, [2049, 1500], span=128, seed=cap + mode, max_pieces=cap, monkeypatch=monkeypatch)


def test_attention_tokens_ctx_32768():
    _attn_case(KV.QUANT_I8, 4, 28, 4, [32768], span=128, seed=3)


@pytest.mark.parametrize("mode", MODES)
def test_q_len_1_bit_identical_and_rows_match_single_token(mode):
    """q_len = 1 reproduces b2_span_attn_run bit for bit; row t of a T-token run matches a single-token run at length
    new_len - T + 1 + t up to fp32 reordering (one bf16 ulp)."""
    from b200spark import ops
    nH, nG, T = 28, 4, 4
    lens = [5, 300, 2049]
    B = len(lens)
    cache, _, _ = _filled_cache(mode, lens, nH, nG, 16, torch.bfloat16, 11 + mode, max(lens) + 1)
    attn = ops.SpanAttn(cache.cfg, B * T)
    ws = ops.Workspace()
    rng = np.random.default_rng(12)
    q = _rand(rng, (B * T, nH * 128), torch.bfloat16)
    nl = torch.tensor(lens, dtype=torch.int32, device="cuda")
    q1 = q.view(B, T, -1)[:, -1].contiguous()
    assert torch.equal(attn.run_tokens(q1, cache, nl, 1, max(lens) + 1, ws), attn(q1, cache, nl, max(lens) + 1, ws))
    multi = attn.run_tokens(q, cache, nl, T, max(lens) + 1, ws).view(B, T, -1).float()
    for t in range(T):
        single = attn(q.view(B, T, -1)[:, t].contiguous(), cache, nl - T + 1 + t, max(lens) + 1, ws).float()
        assert torch.all((multi[:, t] - single).abs() <= 2.0 ** -7 * single.abs() + 1e-5), t


def test_limits():
    from b200spark import _lib, ops
    nH, nG = 28, 4
    cache = ops.SpanCache(2, 64, nH, nG, 16, KV.QUANT_NONE)
    attn = ops.SpanAttn(cache.cfg, 8)
    ws = ops.Workspace()
    q = torch.zeros(2 * 8, nH * 128, dtype=torch.bfloat16, device="cuda")
    nl = torch.full((2,), 20, dtype=torch.int32, device="cuda")
    with pytest.raises(_lib.B2Error, match="LIMIT"):
        attn.run_tokens(q, cache, nl, 8, 64, ws)  # batch * q_len = 16 > max_batch 8
    with pytest.raises(_lib.B2Error, match="LIMIT"):
        attn.run_tokens(q[:17], cache, nl[:1], 17, 64, ws)  # q_len 17
    # head 64: the multi-token kernels are head 128 only
    c64 = ops.SpanCache(2, 64, 14, 2, 16, KV.QUANT_NONE, head=64)
    a64 = ops.SpanAttn(c64.cfg, 8)
    q64 = torch.zeros(2 * 4, 14 * 64, dtype=torch.bfloat16, device="cuda")
    with pytest.raises(_lib.B2Error, match="UNSUPPORTED"):
        a64.run_tokens(q64, c64, nl, 4, 64, ws)


# ------------------------------------------------------------------------------------------------------------- accept
def test_spec_accept_kernel():
    from b200spark import ops
    rng = np.random.default_rng(5)
    B, T = 64, 6
    pred = rng.integers(0, 4, (B, T))
    tokens = rng.integers(0, 4, (B, T))
    tokens[::3, 1:] = pred[::3, :-1]  # every third sequence: all drafts right
    n_ref, nxt_ref = S.accept(tokens, pred)
    tk = torch.from_numpy(tokens).cuda()
    pr = torch.from_numpy(pred).cuda()
    old = torch.arange(B, dtype=torch.int32, device="cuda") + 10
    new = torch.zeros(B, dtype=torch.int32, device="cuda")
    acc = torch.zeros(B, dtype=torch.int32, device="cuda")
    nxt = torch.zeros(B, dtype=torch.int64, device="cuda")
    ops.spec_accept(acc, nxt, old, new, tk, pr)
    torch.cuda.synchronize()
    assert acc.cpu().numpy().tolist() == n_ref.tolist()
    assert nxt.cpu().numpy().tolist() == nxt_ref.tolist()
    assert tk[:, 0].cpu().numpy().tolist() == nxt_ref.tolist() and torch.equal(tk[:, 1:].cpu(), torch.from_numpy(tokens[:, 1:]))
    want_old = np.arange(B) + 10 + n_ref
    assert old.cpu().numpy().tolist() == want_old.tolist() and new.cpu().numpy().tolist() == (want_old + T).tolist()


# ------------------------------------------------------------------------------------------------------------- decode stack
def _greedy(cfg, B, steps, first, **kw):
    """A q_len = 1 stack's greedy continuation: ids [B, steps] and the logits of each step"""
    from b200spark import model
    st = model.DecodeStack(cfg, B, 64, **kw)
    ids, logits = [], []
    cur = first.cuda()
    for _ in range(steps):
        st.ids.copy_(cur)
        cur = st.step().clone()
        ids.append(cur.cpu())
        logits.append(st.logits.float().cpu().clone())
    return torch.stack(ids, 1), logits


def _check_rows(st, pred, B, T, done, live, ref_ids, ref_logits, tol_scale, rows):
    """Rows t < rows of sequence b are single-token steps done[b] + t.  Their logits must lie within the bound of the
    single-token stack's, and their greedy token must equal its token wherever that token's top-2 margin exceeds twice the
    measured logit difference (then no difference of that size can flip it).  A smaller margin is a coin flip, and past it
    the two stacks may continue differently: the sequence is no longer checked (live[b] = False).  Returns the number of
    rows whose token was checked, per sequence."""
    logits = st.logits.float().cpu().view(B, T, -1)
    checked = [0] * B
    for b in range(B):
        for t in range(rows[b]):
            if not live[b] or done[b] + t >= len(ref_logits):
                break
            rl = ref_logits[done[b] + t][b]
            err = (logits[b, t] - rl).abs().max().item()
            assert err <= tol_scale * rl.abs().max().item(), (b, t, err)
            top2 = torch.topk(rl, 2).values
            if (top2[0] - top2[1]).item() <= 2 * err:
                live[b] = False
                break
            assert pred[b, t].item() == ref_ids[b, done[b] + t].item(), (b, t)
            checked[b] += 1
    return checked


@pytest.mark.parametrize("wbits,kv", [(4, "none"), (8, "none"), (4, "i8"), (4, "u4"), (4, "fp8")])
@pytest.mark.parametrize("B", [2, 3])
def test_decode_stack_verify_steps(wbits, kv, B):
    """Verify steps of T = 4 tokens against a single-token stack on the same weights (rows go through the GEMMs at
    M = B*T instead of B, so logits differ by rounding).  Logits within 1e-2 max|logit| (the test_model_gpu.py rule; widened
    to 4e-2 for the uint4 and fp8 caches, where a 1-ulp bf16 difference in a K/V row moves a code by a whole step); tokens
    equal wherever the margin decides them (_check_rows)."""
    from b200spark import model
    T, rounds = 4, 3
    kw = dict(wbits=wbits, kv=kv, span=16, seed=77)
    first = torch.tensor([3, 41, 777][:B], dtype=torch.int64)
    ref_ids, ref_logits = _greedy(model.TINY, B, T * (rounds + 2), first, **kw)
    tol_scale = 4e-2 if kv in ("u4", "fp8") else 1e-2
    # drafts = the single-token stack's own continuation: while the tokens are decided every step accepts all T; eager and
    # graph replay agree bit for bit
    outs, total = {}, 0
    for graph in (False, True):
        st = model.DecodeStack(model.TINY, B, 64, q_len=T, **kw)
        st.tokens[:, 0] = first.cuda()
        done, live, logs = [0] * B, [True] * B, []
        for r in range(rounds):
            for b in range(B):
                st.tokens[b, 1:] = ref_ids[b, done[b]:done[b] + T - 1].cuda()
            if graph and st.graph is None:
                st.capture()
            pred, acc = st.step()
            pred, acc = pred.cpu(), acc.cpu()
            logs.append(st.logits.float().cpu().clone())
            checked = _check_rows(st, pred, B, T, done, live, ref_ids, ref_logits, tol_scale, [T] * B)
            total += sum(checked)
            for b in range(B):
                if checked[b] == T:
                    assert acc[b].item() == T, (r, b, acc)
                done[b] += int(acc[b])
        assert st.lens_old.cpu().tolist() == done
        outs[graph] = torch.stack(logs)
    assert torch.equal(outs[False], outs[True]), "graph replay is bit-identical to eager"
    assert total >= 2 * T * B, total  # on average at least one whole verify step per sequence and run was decided and checked
    # drafts corrupted at chosen positions: the accepted counts and lengths follow the CPU rule on the step's predictions;
    # while the tokens are decided, the accepted count is the corruption point and the emitted tokens are greedy
    st = model.DecodeStack(model.TINY, B, 64, q_len=T, **kw)
    st.tokens[:, 0] = first.cuda()
    done, live = [0] * B, [True] * B
    for r in range(rounds + 2):
        drafts = torch.stack([ref_ids[b, done[b]:done[b] + T - 1] for b in range(B)])
        wrong = (r + np.arange(B)) % T  # 0: nothing corrupted; i: draft i is wrong
        for b in range(B):
            if wrong[b]:
                drafts[b, wrong[b] - 1] = (drafts[b, wrong[b] - 1] + 1) % model.TINY.vocab
        st.tokens[:, 1:] = drafts.cuda()
        tokens = st.tokens.cpu().numpy().copy()
        pred, acc = st.step()
        pred, acc = pred.cpu(), acc.cpu()
        n_ref, _ = S.accept(tokens, pred.numpy())
        assert acc.tolist() == n_ref.tolist()
        want = [int(w) if w else T for w in wrong]
        checked = _check_rows(st, pred, B, T, done, live, ref_ids, ref_logits, tol_scale, want)
        for b in range(B):
            if checked[b] == want[b]:
                assert acc[b].item() == want[b], (r, b, acc)
            done[b] += int(acc[b])
        assert st.lens_old.cpu().tolist() == done and st.lens_new.cpu().tolist() == [L + T for L in done]


# ------------------------------------------------------------------------------------------------------------- needles
# tests/attn_needles.py building blocks: one token per needle carries O(1) of its head's softmax weight.  Every token of a
# sequence shares one query row (the T rows of a sequence differ only in their limits), so a needle at token j must show in
# rows t with j <= new_len - T + t and must not in the others: the T newest tokens carry needles (each row's own token is
# the token just past the limit of the row before it), as do the tile, span and split-KV piece edges.
def _grid_tokens(attn, B, T, max_len, hpg):
    tpb, _ = S.row_blocks(hpg, T)
    per = 2 * 2 * tpb * hpg * (128 + 2) * 4  # two level-0 and two level-1 partial slots of tpb*hpg rows per CTA
    ws = attn.tokens_workspace_bytes(B, T, max_len) - 256
    assert ws > 0 and ws % per == 0, ws
    return ws // per


def _needle_run(mode, dtype, span, nH, nG, T, lens, monkeypatch, max_pieces=None, seed=0, need_piece_edge=False):
    from b200spark import ops
    if max_pieces:
        monkeypatch.setenv("B2_ATTN_MAX_PIECES", str(max_pieces))
    B, hpg, W = len(lens), nH // nG, max(lens)
    prob = A.Problem(lens, nH, nG, 128, dtype, seed)
    cache = ops.SpanCache(B, W, nH, nG, span, mode, dtype=dtype)
    attn = ops.SpanAttn(cache.cfg, B * T)  # after the knobs are set: they are read when the handle is made
    ws = ops.Workspace()
    tpb, nrb = S.row_blocks(hpg, T)
    dec = S.decompose_tokens(lens, T, hpg, nG, _grid_tokens(attn, B, T, W, hpg), max_pieces)
    A.check_decomposition(dec, S.block_lens(lens, T, hpg))
    limits = [[S.row_limit(L, T, t) for t in range(T)] for L in lens]
    per_bg = {}
    edge_at_limit = False
    for b, L in enumerate(lens):
        edges = set()
        for bg in dec.bgs:
            if bg.b // nrb == b:
                edges |= set(A.piece_edges(dec, bg))
                edge_at_limit |= any(pc.tok_lo in limits[b][:-1] for pc in bg.pieces[1:])
        pos = sorted(set(A.tile_and_span_edges(L, span)) | {L - T + t for t in range(T)} | edges)
        for g in range(nG):
            per_bg[(b, g)] = A.schedule(pos, hpg, 4)
    if need_piece_edge:
        assert edge_at_limit, "no split-KV piece starts at a row limit"
    lens_d = torch.tensor(lens, dtype=torch.int32, device="cuda")
    for r in range(max(len(x) for x in per_bg.values())):
        needles = [(b, g * hpg + h, p, 0.0) for (b, g), rr in per_bg.items() if r < len(rr) for h, p in rr[r]]
        k_rows, v_rows, q = prob.rows(needles)
        for b in range(B):
            ops.context_copy(cache, "k", b, torch.from_numpy(k_rows[b].reshape(lens[b], -1)).to(dtype).cuda())
            ops.context_copy(cache, "v", b, torch.from_numpy(v_rows[b].reshape(lens[b], -1)).to(dtype).cuda())
        qd = torch.from_numpy(np.repeat(q[:, None], T, 1).reshape(B * T, -1)).to(dtype).cuda()
        out = attn.run_tokens(qd, cache, lens_d, T, W, ws)
        out2 = attn.run_tokens(qd, cache, lens_d, T, W, ws)
        torch.cuda.synchronize()
        assert torch.equal(out, out2)
        got = out.float().cpu().numpy().reshape(B, T, nH, 128).astype(np.float64)
        assert np.isfinite(got).all()
        kc, ks, vc, vs = [], [], [], []
        for b, L in enumerate(lens):
            nsp = -(-L // span)
            c, s_ = A.from_spans([cache.span_view("k", b, si).cpu().numpy() for si in range(nsp)], mode, span, nG, L, 128, dtype)
            kc.append(c); ks.append(s_)
            c, s_ = A.from_spans([cache.span_view("v", b, si).cpu().numpy() for si in range(nsp)], mode, span, nG, L, 128, dtype)
            vc.append(c); vs.append(s_)
        for t in range(T):
            view = types.SimpleNamespace(lens=[lim[t] for lim in limits], head=128, hpg=hpg, nH=nH, nG=nG, dtype=dtype)
            stale = [(b, h, j) for b, h, j, _ in needles if j >= view.lens[b]]
            res = A.evaluate(view, q, kc, ks, vc, vs, mode, needles, stale=stale)
            assert res.teeth >= A.TEETH, (t, res.teeth, res.weakest)
            assert res.honest <= 1.0, (t, res.honest)
            ratio = np.abs(got[:, t] - res.ref) / res.env
            b, h, d = np.unravel_index(int(np.argmax(ratio)), ratio.shape)
            assert ratio.max() <= 1.0, ("round %d token %d seq %d (limit %d) head %d dim %d" % (r, t, b, view.lens[b], h, d),
                                        float(got[b, t, h, d]), float(res.ref[b, h, d]),
                                        [n for n in needles if n[:2] == (b, h)])


NEEDLE_MODES = [A.NONE, A.I8, A.U4, A.FP8]


@pytest.mark.parametrize("mode", NEEDLE_MODES, ids=lambda m: A.MODE_NAMES[m])
@pytest.mark.parametrize("span", [16, 128])
@pytest.mark.parametrize("nH,nG,T", [(28, 4, 4), (16, 1, 8), (8, 8, 16)])  # 2, 1 and 16 tokens per row block
def test_needles_at_row_limits_tile_and_span_edges(mode, span, nH, nG, T, monkeypatch):
    """The limits of the T rows straddle a tile edge (64 + T/2), a span and tile edge (128 + T/2) and a later one; the
    first sequence is T tokens long, so row 0 sees one token."""
    _needle_run(mode, torch.bfloat16, span, nH, nG, T, [T, 64 + T // 2, 128 + T // 2, 1024 + T // 2], monkeypatch,
                seed=span + T + mode)


@pytest.mark.parametrize("mode", NEEDLE_MODES, ids=lambda m: A.MODE_NAMES[m])
def test_needles_fp16(mode, monkeypatch):
    _needle_run(mode, torch.float16, 16, 28, 4, 4, [4, 66, 130], monkeypatch, seed=50 + mode)


def _len_with_piece_edge_at_limit(T, hpg, nG, grid, cap, lo):
    """A first-sequence length whose T row limits include the first token of a split-KV piece"""
    tpb, nrb = S.row_blocks(hpg, T)
    for L in range(lo, lo + 2000):
        dec = S.decompose_tokens([L, 700], T, hpg, nG, grid, cap)
        lim = {S.row_limit(L, T, t) for t in range(T - 1)}  # first tokens past rows 0 .. T-2
        if any(pc.tok_lo in lim for bg in dec.bgs if bg.b < nrb for pc in bg.pieces[1:]):
            return L
    raise AssertionError("no length found")


@pytest.mark.parametrize("mode", NEEDLE_MODES, ids=lambda m: A.MODE_NAMES[m])
@pytest.mark.parametrize("cap", [None, 4])  # pieces of one tile (> 16 per item: two-level merge); of ~7 tiles (direct merge)
def test_needles_at_piece_edges(mode, cap, monkeypatch):
    """B2_ATTN_MAX_PIECES sets the piece size; the first sequence's length is chosen so that a piece starts at one of its
    row limits (a row's last visible token ends one piece, the next row's starts the next)."""
    from b200spark import ops
    nH, nG, T = 28, 4, 4
    if cap:
        monkeypatch.setenv("B2_ATTN_MAX_PIECES", str(cap))
    probe = ops.SpanCache(2, 2 * 4096, nH, nG, 128, mode)
    grid = _grid_tokens(ops.SpanAttn(probe.cfg, 2 * T), 2, T, 4096, nH // nG)
    L = _len_with_piece_edge_at_limit(T, nH // nG, nG, grid, cap, 1500)
    _needle_run(mode, torch.bfloat16, 128, nH, nG, T, [L, 700], monkeypatch, max_pieces=cap, seed=60 + mode,
                need_piece_edge=True)
