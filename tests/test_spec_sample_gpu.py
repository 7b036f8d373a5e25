"""GPU: b2_sample_tokens and b2_spec_accept_sampled.

Each row of the step form equals b2_sample on that row at its sequence's parameters and counter offsets[b] + depth(t),
bit for bit, and matches the CPU restatement on exact rows; the sampled accept follows the restated walk and advances
the offsets; greedy settings reproduce greedy verification; over the context-hash oracle the device's speculative loop
emits exactly the device's single-token sampling stream; a captured step replays like eager steps."""
import numpy as np
import pytest
import torch

import glue_ref as G
import sample_ref as SR
import spec_sample_ref as SS
import tree_ref as TR

pytestmark = pytest.mark.gpu


def _u64(a):
    return torch.from_numpy(np.asarray(a, np.uint64).view(np.int64).copy()).cuda()


def _np_u64(t):
    return t.cpu().numpy().view(np.uint64)


def _trees(kind, B, T, rng):
    """parents [B][T] of a tree family (None: the chain form, no parents)"""
    if kind == "none":
        return None
    return [SS.TREES[kind](rng, T) for _ in range(B)]


def _params(B, rng, exact):
    """per-sequence (t, k, p, seeds, offsets): exact temperatures (c = 2^j) or realistic ones, greedy sequences included"""
    if exact:
        t = np.array([[SR.exact_temperature(b % 3), 0.0, SR.exact_temperature(1), -1.0][b % 4] for b in range(B)], np.float32)
    else:
        t = np.array([[0.7, 1.0, 0.0, 1.3][b % 4] for b in range(B)], np.float32)
    k = np.array([[0, 50, 1, 0, 7][b % 5] for b in range(B)], np.int32)
    p = np.array([[1.0, 0.9, 0.5, 1.0, 0.95, 0.0][b % 6] for b in range(B)], np.float32)
    seeds = rng.integers(0, 2 ** 63, B, dtype=np.uint64) * np.uint64(2) + np.uint64(1)
    offs = rng.integers(0, 2 ** 63, B, dtype=np.uint64)
    offs[:2] = [2 ** 32 - 2, 2 ** 64 - 3][:min(2, B)]
    return t, k, p, seeds, offs


def _rows(n, R, dt, rng, exact, params, T):
    x = np.empty((R, n), np.float32)
    for r in range(R):
        if exact:
            tb = params[0][r // T]
            j = int(round(np.log2(SR.LOG2E_F32 / tb))) if tb > 0 else 1
            x[r] = SR.exact_row(n, j, 0.0 if r % 2 else 2.0, rng, dt, neg_inf=2 if r % 3 == 0 else 0)
        else:
            v = rng.standard_normal(n) * (1.0 + r % 3)
            v[rng.integers(0, n, 5)] += 8.0
            x[r] = G.ft_values(v, dt)
    return x


def _per_row(lg, T, params, parents):
    """b2_sample on every row alone: its sequence's parameters, offset offsets[b] + depth(t)"""
    from b200spark import ops
    t, k, p, seeds, offs = params
    B = lg.shape[0] // T
    ctr = SS.counters(offs, parents, B, T).reshape(-1)
    idx = np.repeat(np.arange(B), T)
    off = _u64(ctr)
    ids = ops.sample(lg, torch.from_numpy(t[idx]).cuda(), torch.from_numpy(k[idx]).cuda(), torch.from_numpy(p[idx]).cuda(),
                     _u64(seeds[idx]), off)
    return ids.cpu().numpy()


def _tokens_call(lg, T, params, parents):
    from b200spark import ops
    t, k, p, seeds, offs = params
    off = _u64(offs)
    par = None if parents is None else torch.tensor(parents, dtype=torch.int32, device="cuda")
    ids = ops.sample_tokens(lg, T, torch.from_numpy(t).cuda(), torch.from_numpy(k).cuda(), torch.from_numpy(p).cuda(),
                            _u64(seeds), off, parents=par)
    torch.cuda.synchronize()
    assert np.array_equal(_np_u64(off), offs)  # read, not written
    return ids.cpu().numpy()


CASES = [(1, 1), (1, 16), (3, 2), (3, 4), (64, 1), (64, 2)]
BIG = [(1, 16), (3, 4), (64, 1)]


@pytest.mark.parametrize("n", [1, 1000, 32768, 32769, 152064, 262144])
@pytest.mark.parametrize("dt", ["bf16", "fp16"])
@pytest.mark.parametrize("exact", [True, False])
def test_rows_equal_b2_sample(n, dt, exact):
    """every row equals b2_sample on that row at offsets[b] + depth(t), for every tree family; offsets unchanged"""
    ft = G.FTS[dt]
    rng = np.random.default_rng(n + 7 * exact)
    for ci, (B, T) in enumerate(BIG if n > 32769 else CASES + [(64, 16)] * (n == 1000)):
        params = _params(B, rng, exact)
        lg = G.to_ft(_rows(n, B * T, ft, rng, exact, params, T), ft).cuda()
        for kind in (["none", "chain", "star", "random_tree", "deepest_last", "topk"] if T > 1 else ["none"]):
            parents = _trees(kind, B, T, rng)
            got = _tokens_call(lg, T, params, parents)
            assert np.array_equal(got, _per_row(lg, T, params, parents)), (B, T, kind)
        if T == 1:  # q_len = 1: b2_sample's ids
            from b200spark import ops
            t, k, p, seeds, offs = params
            want = ops.sample(lg, *[torch.from_numpy(a).cuda() for a in (t, k, p)], _u64(seeds), _u64(offs)).cpu().numpy()
            assert np.array_equal(_tokens_call(lg, 1, params, None), want)


@pytest.mark.parametrize("n", [4097, 152064])
@pytest.mark.parametrize("dt", ["bf16", "fp16"])
def test_exact_rows_equal_restatement(n, dt):
    """on exact rows the draws equal spec_sample_ref.sample_tokens bit for bit (chains and trees)"""
    ft = G.FTS[dt]
    rng = np.random.default_rng(n)
    for B, T, kind in ((3, 4, "none"), (2, 8, "random_tree"), (2, 6, "topk"), (1, 16, "deepest_last")):
        params = _params(B, rng, True)
        x = _rows(n, B * T, ft, rng, True, params, T)
        parents = _trees(kind, B, T, rng)
        want = SS.sample_tokens(x, T, params[:4], params[4], None if parents is None else np.asarray(parents), form="exact")
        got = _tokens_call(G.to_ft(x, ft).cuda(), T, params, parents)
        assert np.array_equal(got.reshape(B, T), want), (B, T, kind)


def _accept_inputs(B, T, rng, tree):
    pred = rng.integers(0, 50, (B, T))
    par = [TR.random_tree(rng, T) if tree else TR.chain(T) for _ in range(B)]
    tokens = rng.integers(0, 50, (B, T))
    for b in range(B):  # make a share of the drafts right: children copy their parent's draw
        for c in range(1, T):
            if rng.random() < 0.6:
                tokens[b, c] = pred[b, TR.parent(par[b], c)]
    return tokens, pred, par


def _accept_call(tokens, pred, par, offs, lens, sampled=True):
    from b200spark import ops
    B, T = tokens.shape
    d = dict(acc=torch.zeros(B, dtype=torch.int32, device="cuda"), nxt=torch.zeros(B, dtype=torch.int64, device="cuda"),
             old=torch.tensor(lens, dtype=torch.int32, device="cuda"), new=torch.zeros(B, dtype=torch.int32, device="cuda"),
             tk=torch.tensor(tokens, dtype=torch.int64, device="cuda"),
             path=torch.full((B, T), -1, dtype=torch.int32, device="cuda") if par is not None else None,
             off=_u64(offs) if sampled else None)
    ops._spec_accept(d["acc"], d["nxt"], d["old"], d["new"], d["tk"], torch.tensor(pred, dtype=torch.int64, device="cuda"),
                     d["path"], None if par is None else torch.tensor(par, dtype=torch.int32, device="cuda"), d["off"])
    torch.cuda.synchronize()
    return {k: (None if v is None else v.cpu().numpy()) for k, v in d.items()}


@pytest.mark.parametrize("T", [2, 8, 16])
@pytest.mark.parametrize("tree", [False, True])
def test_accept_sampled_equals_restatement(T, tree):
    rng = np.random.default_rng(T + 100 * tree)
    B = 300
    tokens, pred, par = _accept_inputs(B, T, rng, tree)
    offs = rng.integers(0, 2 ** 64 - 32, B, dtype=np.uint64)
    lens = rng.integers(0, 1000, B)
    parents = np.asarray(par) if tree else None
    out = _accept_call(tokens, pred, parents, offs, lens)
    n, paths, nxt = SS.accept(tokens, pred, parents)
    assert np.array_equal(out["acc"], n) and np.array_equal(out["nxt"], nxt) and np.array_equal(out["tk"][:, 0], nxt)
    assert np.array_equal(out["tk"][:, 1:], tokens[:, 1:])
    assert np.array_equal(out["old"], lens + n) and np.array_equal(out["new"], lens + n + T)
    assert np.array_equal(out["off"].view(np.uint64), SS.advance(offs, n, T))
    if tree:
        for b in range(B):
            assert list(out["path"][b, :n[b]]) == paths[b] and np.all(out["path"][b, n[b]:] == -1)
    assert n.max() > 1 and n.min() == 1


@pytest.mark.parametrize("tree", [False, True])
def test_greedy_settings_equal_greedy_verification(tree):
    """temperature <= 0 everywhere: the draws are the argmax ids, and every output of the sampled accept but the offsets
    equals b2_spec_accept / b2_spec_accept_tree on them; the offsets advance by the accepted counts"""
    from b200spark import ops
    rng = np.random.default_rng(3 + tree)
    B, T, n = 8, 8, 32000
    params = list(_params(B, rng, False))
    params[0] = np.array([0.0, -1.0, -0.0, np.nan] * 2, np.float32)
    lg = G.to_ft(_rows(n, B * T, torch.bfloat16, rng, False, params, T), torch.bfloat16).cuda()
    parents = _trees("random_tree" if tree else "none", B, T, rng)
    pred = _tokens_call(lg, T, params, parents).reshape(B, T)
    assert np.array_equal(pred.reshape(-1), ops.argmax(lg).cpu().numpy())
    tokens = pred.copy()
    tokens[:, 1:] = np.roll(pred, 1, axis=1)[:, 1:]  # chains: every draft right
    tokens[::3, 2:] = 7
    lens = np.arange(B) * 5
    par = None if parents is None else np.asarray(parents)
    got = _accept_call(tokens, pred, par, params[4], lens)
    want = _accept_call(tokens, pred, par, params[4], lens, sampled=False)
    for k in ("acc", "nxt", "old", "new", "tk", "path"):
        assert (got[k] is None and want[k] is None) or np.array_equal(got[k], want[k]), k
    assert np.array_equal(got["off"].view(np.uint64), params[4] + got["acc"].astype(np.uint64))


# ------------------------------------------------------------------------------------------------------------- streams
def _single_stream(oracle, prompts, params, L):
    """b2_sample one token per step over the oracle's rows"""
    from b200spark import ops
    t, k, p, seeds, offs = params
    B = len(prompts)
    ctx = [list(pr) for pr in prompts]
    dev = [torch.from_numpy(a).cuda() for a in (t, k, p)] + [_u64(seeds)]
    off = _u64(offs)
    for _ in range(L):
        lg = G.to_ft(np.stack([oracle.row(c) for c in ctx]), oracle.dt).cuda()
        ids = ops.sample(lg, *dev, off).cpu().numpy()
        for b in range(B):
            ctx[b].append(int(ids[b]))
    return [c[len(pr):] for c, pr in zip(ctx, prompts)], _np_u64(off)


def _spec_stream(oracle, prompts, params, L, T, tree, drafter, truths, seed):
    """b2_sample_tokens + b2_spec_accept_sampled over the oracle's rows"""
    from b200spark import ops
    t, k, p, seeds, offs = params
    B = len(prompts)
    rng = np.random.default_rng(seed)
    ctx = [list(pr) for pr in prompts]
    out = [[] for _ in range(B)]
    dev = [torch.from_numpy(a).cuda() for a in (t, k, p)] + [_u64(seeds)]
    off = _u64(offs)
    acc, nxt = torch.zeros(B, dtype=torch.int32, device="cuda"), torch.zeros(B, dtype=torch.int64, device="cuda")
    old, new = torch.zeros(B, dtype=torch.int32, device="cuda"), torch.zeros(B, dtype=torch.int32, device="cuda")
    path = torch.zeros(B, T, dtype=torch.int32, device="cuda")
    dor = SS.Oracle(oracle.vocab, oracle.seed, oracle.dt, perturb=0.7) if drafter == "sampled" else None
    steps = accepted = 0
    while min(len(o) for o in out) < L:
        pars = [SS.TREES[tree](rng, T) for _ in range(B)]
        tokens = np.stack([SS.draft(drafter, rng, oracle, ctx[b], pars[b], truths[b][len(out[b]):], dor) for b in range(B)])
        lg = G.to_ft(np.stack([oracle.row(c) for b in range(B) for c in SS.contexts(ctx[b], tokens[b], pars[b])]), oracle.dt).cuda()
        par = None if tree == "chain" else torch.tensor(pars, dtype=torch.int32, device="cuda")
        pred = ops.sample_tokens(lg, T, *dev, off, parents=par).view(B, T)
        tk = torch.from_numpy(tokens).cuda()
        ops._spec_accept(acc, nxt, old, new, tk, pred, path if par is not None else None, par, off)
        pred, n, pa = pred.cpu().numpy(), acc.cpu().numpy(), path.cpu().numpy()
        for b in range(B):
            emitted = [int(pred[b, pa[b, i] if par is not None else i]) for i in range(n[b])]
            out[b] += emitted
            ctx[b] += emitted
        assert np.array_equal(tk[:, 0].cpu().numpy(), [ctx[b][-1] for b in range(B)])
        steps += 1
        accepted += int(n.sum())
    return out, _np_u64(off), accepted / (steps * B)


@pytest.mark.parametrize("vocab", [4096, 152064])
def test_stream_equality_on_device(vocab):
    """the device's speculative loop emits the device's single-token stream, for every drafter and tree family, and ends
    at the same offsets"""
    oracle = SS.Oracle(vocab, seed=vocab)
    B, L = 4, 12
    prompts = [[b + 1, 5 * b + 2, 9] for b in range(B)]
    params = _params(B, np.random.default_rng(vocab), False)
    Ts = [2, 4, 8, 16] if vocab == 4096 else [8]
    truths, _ = _single_stream(oracle, prompts, params, L * max(Ts))  # a step emits at most T tokens
    rates = {}
    for T in Ts:
        for tree in SS.TREES:
            for drafter in SS.DRAFTERS:
                out, off, rate = _spec_stream(oracle, prompts, params, L, T, tree, drafter, truths, seed=T)
                for b in range(B):
                    assert out[b] == truths[b][:len(out[b])], (T, tree, drafter, b)
                    assert int(off[b]) == (int(params[4][b]) + len(out[b])) % 2 ** 64, (T, tree, drafter, b)
                rates[(T, tree, drafter)] = rate
    assert max(r for (T, tr, d), r in rates.items() if d == "truth") > 1.5, rates


def test_graph_replay():
    """sample_tokens + the sampled accept captured once and replayed 8 times, drafts and rows rewritten between replays,
    equal 8 eager steps: ids, accepted counts, paths and offsets"""
    from b200spark import ops
    rng = np.random.default_rng(8)
    B, T, n = 3, 6, 152064
    params = _params(B, rng, False)
    dev = [torch.from_numpy(a).cuda() for a in params[:3]] + [_u64(params[3])]
    rows = [G.to_ft(_rows(n, B * T, torch.bfloat16, rng, False, params, T), torch.bfloat16).cuda() for _ in range(8)]
    drafts = [torch.from_numpy(rng.integers(0, 30, (B, T - 1))).cuda() for _ in range(8)]
    par = torch.tensor([SS.TREES["random_tree"](rng, T) for _ in range(B)], dtype=torch.int32, device="cuda")
    st = dict(lg=torch.empty_like(rows[0]), pred=torch.zeros(B * T, dtype=torch.int64, device="cuda"),
              tk=torch.zeros(B, T, dtype=torch.int64, device="cuda"), acc=torch.zeros(B, dtype=torch.int32, device="cuda"),
              nxt=torch.zeros(B, dtype=torch.int64, device="cuda"), old=torch.zeros(B, dtype=torch.int32, device="cuda"),
              new=torch.zeros(B, dtype=torch.int32, device="cuda"), path=torch.zeros(B, T, dtype=torch.int32, device="cuda"),
              off=_u64(params[4]))

    def step():
        ops.sample_tokens(st["lg"], T, *dev, st["off"], parents=par, out=st["pred"])
        ops._spec_accept(st["acc"], st["nxt"], st["old"], st["new"], st["tk"], st["pred"].view(B, T), st["path"], par, st["off"])

    def feed(i):
        st["lg"].copy_(rows[i])
        st["tk"][:, 1:] = drafts[i]

    def run(replay):
        for k in ("tk", "acc", "old", "new", "path", "pred"):
            st[k].zero_()
        st["off"].copy_(_u64(params[4]))
        outs = []
        for i in range(8):
            feed(i)
            replay() if replay else step()
            torch.cuda.synchronize()
            outs.append([st[k].clone() for k in ("pred", "acc", "path", "off", "old", "tk")])
        return outs

    eager = run(None)
    step()  # warm-up, then capture
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        step()
    replayed = run(g.replay)
    for i in range(8):
        for a, b in zip(eager[i], replayed[i]):
            assert torch.equal(a, b), i
