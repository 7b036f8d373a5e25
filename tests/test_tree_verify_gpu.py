"""GPU: tree-structured speculative verification — draft-tree append, attention with per-row ancestor masks, greedy tree
acceptance on the device, compaction of the accepted path, and the decode stack's tree verify step.

Attention is checked against fp64 attention (tests/tree_ref.py) over the cache bytes read back from the device, with the
bound of test_spec_decode_gpu.py: 2e-3 + 2^-7 |ref| (fp16 output 2^-9), plus the rounding of the probabilities,
u_P sum_j p_j |V_j|, for rows that see at most one tile.  Chains must reproduce the multi-token entry points bit for bit."""
import numpy as np
import pytest
import torch

import attn_needles as A
import tree_ref as TR
from oracle import kvcache_ref as KV

pytestmark = pytest.mark.gpu

MODES = [0, 1, 2, 3]  # none, i8, u4, fp8


def _rand(rng, shape, dtype):
    return torch.from_numpy(rng.standard_normal(shape).astype(np.float32)).to(dtype).cuda()


def _parents(trees):
    return torch.tensor(trees, dtype=torch.int32, device="cuda")


class _Dense:
    """.dense(b, L) of a device cache: the values its span bytes hold (attn_needles.from_spans), for tree_ref"""

    def __init__(self, cache, which, mode, dtype, lens):
        self.n_groups, self.head = cache.cfg.n_groups, 128
        self.vals = []
        for b, L in enumerate(lens):
            spans = [cache.span_view(which, b, si).cpu().numpy() for si in range(-(-L // cache.cfg.span_len))]
            c, s = A.from_spans(spans, mode, cache.cfg.span_len, self.n_groups, L, 128, dtype)
            self.vals.append(c * s[..., None])

    def dense(self, b, length):
        return self.vals[b][:, :length]


def _check(got, ref, ref_abs, lens, trees, mode, dtype):
    """got / ref / ref_abs [B, T, nH, 128]; rows that see at most one tile add u_P sum_j p_j |V_j|"""
    err = np.abs(got - ref)
    bound = 2e-3 + (2.0 ** -9 if dtype == torch.float16 else 2.0 ** -7) * np.abs(ref)
    u_p, _ = A.p_type(mode, dtype, 128)
    seen = np.array([TR.tree_mask(L, par).sum(1) for L, par in zip(lens, trees)])  # [B, T] tokens each row sees
    bound = bound + np.where(seen <= A.TILE, u_p, 0.0)[:, :, None, None] * ref_abs
    assert np.all(np.isfinite(got))
    worst = np.unravel_index(int(np.argmax(err - bound)), err.shape)
    assert np.all(err <= bound), ("seq %d node %d head %d dim %d" % worst, float(err[worst]), float(bound[worst]))


def _trees(kind, T, B, rng):
    make = {"chain": lambda: TR.chain(T), "star": lambda: TR.star(T), "deepest_last": lambda: TR.deepest_last(T),
            "random": lambda: TR.random_tree(rng, T)}[kind]
    return [make() for _ in range(B)]


# ---------------------------------------------------------------------------------------------------------------- append
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("span", [16, 128])
@pytest.mark.parametrize("rope", [False, True])
def test_append_tree(mode, dtype, span, rope):
    """Chain parents: the bytes of b2_span_cache_append_tokens.  Random trees: row t's bytes at slot old + t equal a single
    append of the same qkv row at position old + depth(t)."""
    from b200spark import ops
    rng = np.random.default_rng(span + mode + (7 if rope else 0) + (3 if dtype == torch.float16 else 0))
    nH, nG, T = 8, 2, 7
    old = [0, 13, span - 2, 2 * span - 1]  # ragged, crossing span boundaries
    B = len(old)
    r = (1e6, 128) if rope else None
    old_d = torch.tensor(old, dtype=torch.int32, device="cuda")
    qkv = _rand(rng, (B * T, (nH + 2 * nG) * 128), dtype)
    # chain
    a = ops.SpanCache(B, 3 * span, nH, nG, span, mode, fill=0xFF, dtype=dtype)
    c = ops.SpanCache(B, 3 * span, nH, nG, span, mode, fill=0xFF, dtype=dtype)
    q_tree = ops.cache_append_tree(a, qkv, old_d, _parents([TR.chain(T)] * B), T, rope=r)
    q_tok = ops.cache_append_tokens(c, qkv, old_d, T, rope=r)
    torch.cuda.synchronize()
    assert torch.equal(a.k_pool, c.k_pool) and torch.equal(a.v_pool, c.v_pool)
    assert torch.equal(q_tree.view(torch.int16), q_tok.view(torch.int16))
    # random trees
    trees = [TR.random_tree(rng, T) for _ in range(B)]
    t_cache = ops.SpanCache(B, 3 * span, nH, nG, span, mode, fill=0xFF, dtype=dtype)
    q_tree = ops.cache_append_tree(t_cache, qkv, old_d, _parents(trees), T, rope=r).view(B, T, -1)
    depth = [TR.depth_anc(par)[0] for par in trees]
    rows = qkv.view(B, T, -1)
    for t in range(T):
        s = ops.SpanCache(B, 3 * span, nH, nG, span, mode, fill=0xFF, dtype=dtype)
        pos = torch.tensor([old[b] + depth[b][t] for b in range(B)], dtype=torch.int32, device="cuda")
        q1 = ops.cache_append(s, rows[:, t].contiguous(), pos, rope=r)
        torch.cuda.synchronize()
        assert torch.equal(q_tree[:, t].view(torch.int16), q1.view(torch.int16)), t
        for b in range(B):
            src, dst = int(pos[b]), old[b] + t
            for which in ("k", "v"):
                sv = s.span_view(which, b, src // span).cpu().numpy()
                tv = t_cache.span_view(which, b, dst // span).cpu().numpy()
                for g in range(nG):
                    for (s0, s1), (d0, d1) in zip(TR.row_ranges(mode, span, nG, g, src % span), TR.row_ranges(mode, span, nG, g, dst % span)):
                        assert np.array_equal(sv[s0:s1], tv[d0:d1]), (t, b, which, g)


# ------------------------------------------------------------------------------------------------------------- attention
def _filled_cache(mode, lens, nH, nG, span, dtype, seed, max_len):
    from b200spark import ops
    rng = np.random.default_rng(seed)
    cache = ops.SpanCache(len(lens), max_len, nH, nG, span, mode, fill=0xFF, dtype=dtype)
    for b, L in enumerate(lens):
        ops.context_copy(cache, "k", b, _rand(rng, (L, nG * 128), dtype))
        ops.context_copy(cache, "v", b, _rand(rng, (L, nG * 128), dtype))
    torch.cuda.synchronize()
    return cache


def _tree_case(mode, T, nH, nG, lens, kind, span=16, dtype=torch.bfloat16, seed=0, max_pieces=None, monkeypatch=None):
    from b200spark import ops
    max_len = max(lens) + 1
    cache = _filled_cache(mode, lens, nH, nG, span, dtype, seed, max_len)
    if max_pieces is not None:
        monkeypatch.setenv("B2_ATTN_MAX_PIECES", str(max_pieces))
    attn = ops.SpanAttn(cache.cfg, len(lens) * T)
    rng = np.random.default_rng(seed + 1)
    trees = _trees(kind, T, len(lens), rng)
    q = _rand(rng, (len(lens) * T, nH * 128), dtype)
    new_lens = torch.tensor(lens, dtype=torch.int32, device="cuda")
    par = _parents(trees)
    ws = ops.Workspace()
    out = attn.run_tree(q, cache, new_lens, par, T, max_len, ws)
    out2 = attn.run_tree(q, cache, new_lens, par, T, max_len, ws)
    torch.cuda.synchronize()
    assert torch.equal(out, out2), "deterministic, counters re-armed"
    kd, vd = _Dense(cache, "k", mode, dtype, lens), _Dense(cache, "v", mode, dtype, lens)
    ref, ref_abs = TR.attention_tree(q.float().cpu().numpy().reshape(len(lens), T, nH, 128), kd, vd, lens, trees, T, nH,
                                     1 / np.sqrt(128), with_abs=True)
    _check(out.float().cpu().numpy().reshape(len(lens), T, nH, 128), ref, ref_abs, lens, trees, mode, dtype)
    if kind == "chain":
        tok = attn.run_tokens(q, cache, new_lens, T, max_len, ws)
        torch.cuda.synchronize()
        assert torch.equal(out.view(torch.int16), tok.view(torch.int16)), "a chain is bit-identical to run_tokens"


@pytest.mark.parametrize("kind", ["random", "star", "chain", "deepest_last"])
@pytest.mark.parametrize("T", [2, 4, 8, 16])
@pytest.mark.parametrize("nH,nG", [(8, 8), (16, 4), (28, 4), (16, 2), (16, 1)])  # hpg 1, 4, 7, 8, 16
def test_attention_tree_bf16(kind, T, nH, nG):
    _tree_case(0, T, nH, nG, [T, T + 61, 64 + T, 200, 2049], kind, seed=T * 31 + nH + len(kind))


@pytest.mark.parametrize("mode", MODES[1:])
@pytest.mark.parametrize("kind", ["random", "chain"])
@pytest.mark.parametrize("T", [4, 8, 16])
@pytest.mark.parametrize("nH,nG", [(28, 4), (16, 1)])
def test_attention_tree_quantized(mode, kind, T, nH, nG):
    _tree_case(mode, T, nH, nG, [T, 65, 130, 2049], kind, seed=T + nH + 5 * mode + len(kind))


@pytest.mark.parametrize("mode", MODES)
def test_attention_tree_fp16(mode):
    _tree_case(mode, 8, 28, 4, [8, 100, 700], "random", dtype=torch.float16, seed=40 + mode)


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("cap", [4, 17])
@pytest.mark.parametrize("kind", ["random", "chain"])
def test_attention_tree_piece_caps(mode, cap, kind, monkeypatch):
    """B2_ATTN_MAX_PIECES forcing the direct (<= 16 pieces) and the two-level merge"""
    _tree_case(mode, 8, 28, 4, [2049, 1500], kind, span=128, seed=cap + mode, max_pieces=cap, monkeypatch=monkeypatch)


@pytest.mark.parametrize("kind", ["random", "chain"])
def test_attention_tree_ctx_32768(kind):
    _tree_case(1, 8, 28, 4, [32768], kind, span=128, seed=3)


# ------------------------------------------------------------------------------------------------------------- needles
@pytest.mark.parametrize("mode", MODES, ids=lambda m: A.MODE_NAMES[m])
def test_needle_in_a_draft_slot(mode):
    """A needle (tests/attn_needles.py) for every head at draft slot j: rows with j among their ancestors are dominated
    by it; the other rows (siblings, cousins) equal the output without the needle, within the bound."""
    from b200spark import ops
    nH, nG, T, span, dtype = 8, 2, 8, 16, torch.bfloat16
    hpg = nH // nG
    lens = [T + 5, 64 + T + 3, 200]
    trees = [[0, 0, 0, 1, 1, 2, 3, 5], [0, 0, 1, 2, 0, 4, 4, 6], [0, 0, 0, 0, 1, 2, 3, 4]]
    B, W = len(lens), max(lens)
    prob = A.Problem(lens, nH, nG, 128, dtype, seed=70 + mode)
    cache = ops.SpanCache(B, W, nH, nG, span, mode, dtype=dtype)
    attn = ops.SpanAttn(cache.cfg, B * T)
    ws = ops.Workspace()
    lens_d, par = torch.tensor(lens, dtype=torch.int32, device="cuda"), _parents(trees)
    anc = [TR.depth_anc(p)[1] for p in trees]

    def run(needles):
        k_rows, v_rows, q = prob.rows(needles)
        for b in range(B):
            ops.context_copy(cache, "k", b, torch.from_numpy(k_rows[b].reshape(lens[b], -1)).to(dtype).cuda())
            ops.context_copy(cache, "v", b, torch.from_numpy(v_rows[b].reshape(lens[b], -1)).to(dtype).cuda())
        qd = torch.from_numpy(np.repeat(q[:, None], T, 1).reshape(B * T, -1)).to(dtype).cuda()
        out = attn.run_tree(qd, cache, lens_d, par, T, W, ws)
        torch.cuda.synchronize()
        got = out.float().cpu().numpy().reshape(B, T, nH, 128)
        kd, vd = _Dense(cache, "k", mode, dtype, lens), _Dense(cache, "v", mode, dtype, lens)
        ref, ref_abs = TR.attention_tree(qd.float().cpu().numpy().reshape(B, T, nH, 128), kd, vd, lens, trees, T, nH,
                                         1 / np.sqrt(128), with_abs=True)
        _check(got, ref, ref_abs, lens, trees, mode, dtype)
        return got, ref

    base, base_ref = run([])
    mark = 128 - A.R  # the marker dim of the only needle of a (sequence, kv-head)
    for j in (1, 2, 4, 5):
        # one needle per (sequence, kv-head) at slot j (the builder rewrites the whole K row of its token), head j % hpg
        needles = [(b, g * hpg + j % hpg, lens[b] - T + j, 0.0) for b in range(B) for g in range(nG)]
        got, _ = run(needles)
        for b in range(B):
            for t in range(T):
                if anc[b][t] >> j & 1:  # the needle carries most of its head's weight: the marker dim moves by >= MARK / 2
                    for g in range(nG):
                        h = g * hpg + j % hpg
                        assert got[b, t, h, mark] - base[b, t, h, mark] >= A.MARK / 2, (j, b, t, h, got[b, t, h, mark])
                else:  # the slot is not visible: every head as without the needle
                    env = 2e-3 + 2.0 ** -7 * np.abs(base_ref[b, t]) + 2.0 ** -8
                    assert np.all(np.abs(got[b, t] - base[b, t]) <= env), (j, b, t)


# ------------------------------------------------------------------------------------------------------------- accept
def test_spec_accept_tree_kernel():
    from b200spark import ops
    rng = np.random.default_rng(5)
    B, T = 96, 8
    trees = [TR.random_tree(rng, T) if b % 4 else TR.chain(T) for b in range(B)]
    trees[1] = TR.star(T)
    pred = rng.integers(0, 3, (B, T))
    tokens = rng.integers(0, 3, (B, T))
    for b in range(0, B, 3):  # plant a matching root-to-leaf walk
        u = 0
        while True:
            kids = [c for c in range(u + 1, T) if trees[b][c] == u]
            if not kids:
                break
            c = kids[int(rng.integers(0, len(kids)))]
            tokens[b, c] = pred[b, u]
            u = c
    n_ref, paths_ref, nxt_ref = TR.accept_tree(tokens, pred, trees)
    assert max(n_ref) >= 4
    tk, pr = torch.from_numpy(tokens).cuda(), torch.from_numpy(pred).cuda()
    par = _parents(trees)
    path = torch.full((B, T), -7, dtype=torch.int32, device="cuda")
    old = torch.arange(B, dtype=torch.int32, device="cuda") + 10
    new = torch.zeros(B, dtype=torch.int32, device="cuda")
    acc = torch.zeros(B, dtype=torch.int32, device="cuda")
    nxt = torch.zeros(B, dtype=torch.int64, device="cuda")
    ops.spec_accept_tree(acc, path, nxt, old, new, tk, pr, par)
    torch.cuda.synchronize()
    assert acc.cpu().tolist() == n_ref.tolist()
    path = path.cpu().numpy()
    assert all(path[b, :n_ref[b]].tolist() == paths_ref[b] for b in range(B))
    assert nxt.cpu().tolist() == nxt_ref.tolist() and tk[:, 0].cpu().tolist() == nxt_ref.tolist()
    assert torch.equal(tk[:, 1:].cpu(), torch.from_numpy(tokens[:, 1:]))
    want_old = np.arange(B) + 10 + n_ref
    assert old.cpu().tolist() == want_old.tolist() and new.cpu().tolist() == (want_old + T).tolist()
    # a chain: b2_spec_accept's results
    tk2, old2, new2 = torch.from_numpy(tokens).cuda(), torch.zeros(B, dtype=torch.int32, device="cuda"), torch.zeros(B, dtype=torch.int32, device="cuda")
    acc2, nxt2 = torch.zeros_like(acc), torch.zeros_like(nxt)
    ops.spec_accept(acc2, nxt2, old2, new2, tk2, pr)
    tk3, old3, new3 = torch.from_numpy(tokens).cuda(), torch.zeros_like(old2), torch.zeros_like(new2)
    acc3, nxt3, path3 = torch.zeros_like(acc), torch.zeros_like(nxt), torch.zeros(B, T, dtype=torch.int32, device="cuda")
    ops.spec_accept_tree(acc3, path3, nxt3, old3, new3, tk3, pr, _parents([TR.chain(T)] * B))
    torch.cuda.synchronize()
    for x, y in ((acc2, acc3), (nxt2, nxt3), (old2, old3), (new2, new3), (tk2, tk3)):
        assert torch.equal(x, y)


# ------------------------------------------------------------------------------------------------------------- compaction
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("span", [16, 128])
def test_cache_compact(mode, span):
    """3 layers, one launch: span bytes equal tree_ref.compact per (layer, sequence, K / V); hazard paths, paths across
    span edges, n = 1 and n = T"""
    from b200spark import ops
    rng = np.random.default_rng(mode + span)
    nH, nG, T, layers = 8, 2, 8, 3
    paths = [[0, 2, 3], [0, 2, 3, 4, 5], [0, 3, 5, 6, 7], [0], list(range(T)), [0, 1, 3, 4], [0, 4, 5, 7], [0, 7]]
    B = len(paths)
    base = [span - 2, 0, span - 3, 5, span - 4, 2 * span - 1, 1, span - 7]
    caches = [ops.SpanCache(B, 3 * span, nH, nG, span, mode) for _ in range(layers)]
    for c in caches:
        c.k_pool.copy_(torch.randint(0, 256, c.k_pool.shape, dtype=torch.uint8, generator=torch.Generator().manual_seed(1)).cuda())
        c.v_pool.copy_(torch.randint(0, 256, c.v_pool.shape, dtype=torch.uint8, generator=torch.Generator().manual_seed(2)).cuda())
    torch.cuda.synchronize()
    before = {(li, which, b): [c.span_view(which, b, si).cpu().numpy().copy() for si in range(c.max_spans)]
              for li, c in enumerate(caches) for which in ("k", "v") for b in range(B)}
    n = [len(p) for p in paths]
    path = np.full((B, T), 99, np.int32)  # entries past n are ignored
    for b, p in enumerate(paths):
        path[b, :len(p)] = p
    old = torch.tensor([base[b] + n[b] for b in range(B)], dtype=torch.int32, device="cuda")
    acc = torch.tensor(n, dtype=torch.int32, device="cuda")
    ops.cache_compact(caches, old, acc, torch.from_numpy(path).cuda(), T)
    torch.cuda.synchronize()
    for (li, which, b), spans in before.items():
        TR.compact(spans, mode, span, nG, base[b], paths[b])
        got = [caches[li].span_view(which, b, si).cpu().numpy() for si in range(caches[li].max_spans)]
        for si in range(len(spans)):
            assert np.array_equal(got[si], spans[si]), (li, which, b, si, paths[b])


# ------------------------------------------------------------------------------------------------------------- decode stack
def _ref_decoder(st, kv):
    from oracle import decoder_ref as DR
    if kv == "fp8":
        import kv_fp8_ref as F8
        return F8.decoder_ref(st)
    return DR.from_stack(st, {"none": KV.QUANT_NONE, "i8": KV.QUANT_I8, "u4": KV.QUANT_U4}[kv])


@pytest.mark.parametrize("wbits,kv", [(4, "none"), (8, "none"), (4, "i8"), (4, "u4"), (4, "fp8")])
def test_decode_stack_tree_steps(wbits, kv):
    """Tree verify steps (T = 6): node 0 the last emitted token, a first branch of two wrong drafts (nodes 1, 2) and a second
    branch (nodes 3, 4, 5) holding the oracle's greedy continuation, so the accepted path is [0, 3, 4, 5] and compaction
    moves three rows.  The emitted tokens must be plain greedy decoding by oracle.decoder_ref wherever the top-2 margin
    decides them (test_spec_decode_gpu.py's rule); the cache after compaction must match a single-token stack that decoded
    the same tokens; eager and graph replay agree bit for bit."""
    from b200spark import model
    B, T, rounds = 2, 6, 4
    par = [0, 0, 1, 0, 3, 4]
    kw = dict(wbits=wbits, kv=kv, span=16, seed=77)
    first = torch.tensor([3, 41], dtype=torch.int64)
    st0 = model.DecodeStack(model.TINY, B, 64, keep_ref=True, **kw)
    ref = _ref_decoder(st0, kv)
    ref.reset(B)
    steps = 4 * rounds + 2
    ids, ref_ids, ref_logits = first, [], []
    for t in range(steps):
        rlog, ids = ref.step(ids, [t] * B)
        ref_ids.append(ids.clone())
        ref_logits.append(rlog)
    ref_ids = torch.stack(ref_ids, 1)
    tol_scale = 4e-2 if kv in ("u4", "fp8") else 1e-2
    outs, checked_total = {}, 0
    for graph in (False, True):
        st = model.DecodeStack(model.TINY, B, 64, q_len=T, tree=True, **kw)
        st.tokens[:, 0] = first.cuda()
        st.parents.copy_(torch.tensor([par] * B, dtype=torch.int32))
        done, live, logs, emitted = [0] * B, [True] * B, [], [[int(f)] for f in first]
        for r in range(rounds):
            for b in range(B):
                g = ref_ids[b, done[b]:done[b] + 3]
                st.tokens[b, 1:] = torch.cat([(g[:1] + 1) % model.TINY.vocab, g[:1], g]).cuda()
            if graph and st.graph is None:
                st.capture()
            pred, acc, path = st.step()
            pred, acc, path = pred.cpu(), acc.cpu(), path.cpu()
            logits = st.logits.float().cpu().view(B, T, -1)
            logs.append(logits.clone())
            for b in range(B):
                n = int(acc[b])
                p = path[b, :n].tolist()
                checked = 0
                for i in range(4):  # the nodes of the greedy branch: 0, 3, 4, 5
                    node = [0, 3, 4, 5][i]
                    if not live[b]:
                        break
                    rl = ref_logits[done[b] + i][b]
                    err = (logits[b, node] - rl).abs().max().item()
                    assert err <= tol_scale * rl.abs().max().item(), (r, b, node, err)
                    top2 = torch.topk(rl, 2).values
                    if (top2[0] - top2[1]).item() <= 2 * err:
                        live[b] = False
                        break
                    assert pred[b, node].item() == ref_ids[b, done[b] + i].item(), (r, b, node)
                    checked += 1
                if checked == 4:
                    assert n == 4 and p == [0, 3, 4, 5], (r, b, p)
                checked_total += checked
                emitted[b] += [int(pred[b, u]) for u in p]
                done[b] += n
        assert st.lens_old.cpu().tolist() == done and st.lens_new.cpu().tolist() == [d + T for d in done]
        outs[graph] = torch.stack(logs)
        # the cache: a single-token stack fed the same tokens holds the same rows in slots 0 .. done-1
        one = model.DecodeStack(model.TINY, B, 64, **kw)
        for t in range(max(done)):
            one.ids.copy_(torch.tensor([e[min(t, len(e) - 1)] for e in emitted], dtype=torch.int64))
            one.step()
        torch.cuda.synchronize()
        mode = model.KV_MODES[kv]
        for li in range(len(st.layers)):
            for which in ("k", "v"):
                for b in range(B):
                    L = done[b]
                    got = _Dense(st.layers[li]["cache"], which, mode, st.dtype, [0] * b + [L]).dense(b, L)
                    want = _Dense(one.layers[li]["cache"], which, mode, st.dtype, [0] * b + [L]).dense(b, L)
                    # the rows went through the GEMMs at M = B*T instead of B: rounding differences, compounded over the
                    # layers (layer 1's K rows: up to 1.5 bf16 ulps of the row's largest value measured), within 2e-2 of
                    # the row's max (4e-2 for uint4 / fp8, as for the logits), plus one code step of the quantized modes.
                    # A row left at its node slot, or another node's row, differs by O(1).
                    amax = np.abs(want).max(-1, keepdims=True)
                    step_ = {0: 0.0, 1: 2.0 / 255, 2: 2.0 / 15, 3: 1.0 / 8}[mode] * amax
                    assert np.all(np.abs(got - want) <= 2 * tol_scale * amax + step_), (li, which, b, float(np.abs(got - want).max()))
    assert torch.equal(outs[False], outs[True]), "graph replay is bit-identical to eager"
    assert checked_total >= 2 * 4 * B, checked_total
