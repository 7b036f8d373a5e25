"""GPU: b2_penalize_tokens bit for bit against its restatement (tests/penalty_tokens_ref.py) and against b2_penalize run
on every virtual history loaded into its own slot; q_len = 1, a read-only history, vocab shards and graph replay.

The headline: over the context-hash oracle (spec_sample_ref.Oracle), a penalised speculative loop (drafts, then
penalize_tokens, sample_tokens or argmax, the accept and append_tokens) emits exactly the single-token penalised stream
(penalize, sample or argmax, append), ends at the same offsets and leaves the same history arrays, for every drafter,
chains and trees, greedy and sampled; captured in one CUDA graph, the speculative tail replays like its eager steps."""
import ctypes as C

import numpy as np
import pytest
import torch

import glue_ref as G
import penalty_ref as P
import penalty_tokens_ref as PT
import sample_ref as SR
import spec_sample_ref as SS

pytestmark = pytest.mark.gpu

PAD = 5  # columns n .. n + PAD - 1 of every row hold a sentinel that must survive
SENTINEL = 0x7E11


@pytest.fixture(scope="module")
def ops():
    from b200spark import ops as o
    return o


def upload(x, ft):
    rows, n = x.shape
    t = torch.empty(rows, n + PAD, dtype=P.FTS[ft], device="cuda")
    t.view(torch.int16)[:, n:] = SENTINEL
    t[:, :n] = torch.from_numpy(x).to(P.FTS[ft]).cuda()
    return t


def load_raw(ops, h, slot, ids, prompt_len):
    """b2_history_load without the front end's range check, so stored -1 entries can be loaded as they are"""
    from b200spark import _lib
    t = torch.tensor([int(v) for v in ids] or [0], dtype=torch.int32, device="cuda")
    _lib.check(_lib.lib.b2_history_load(C.byref(h.c), slot, C.c_void_p(t.data_ptr()), len(ids), prompt_len, ops._stream()),
               "b2_history_load")
    torch.cuda.synchronize()


def device_params(ops, prm, rows=None):
    rows = rows or len(prm["repetition"])
    pen = ops.Penalties(rows)
    for k in P.neutral(0):
        getattr(pen, k).copy_(torch.tensor(prm[k]))
    return pen


def make_parents(kind, B, T, rng):
    if kind == "none":
        return None
    if kind == "malformed":  # parents outside [0, t) are read as the root
        return [[int(rng.integers(-3, T + 3)) for _ in range(T)] for _ in range(B)]
    return [SS.TREES[kind](rng, T) for _ in range(B)]


def make_drafts(hists, n, T, rng):
    """[B][T] int64 drafts: copies of the history after an earlier occurrence of its last token (n-gram matches across the
    base / path boundary), a small pool that repeats itself, base ids, and ids outside [0, n)"""
    out = []
    for b, h in enumerate(hists):
        h = [int(v) for v in h]
        row = [int(rng.integers(0, n + 3))] + [int(v) for v in rng.integers(0, n, T - 1)]
        kind = b % 4
        if kind == 0 and len(h) >= 2:
            starts = [j + 1 for j in range(len(h) - 1) if h[j] == h[-1]] or [int(rng.integers(0, len(h)))]
            k = starts[int(rng.integers(0, len(starts)))]
            for i in range(1, T):
                row[i] = h[k + i - 1] if k + i - 1 < len(h) else row[i]
        elif kind == 1:
            pool = rng.integers(0, n, 3)
            row[1:] = [int(pool[int(rng.integers(0, 3))]) for _ in range(T - 1)]
        elif kind == 2 and h:
            row[1:] = [h[int(rng.integers(0, len(h)))] for _ in range(T - 1)]
        bad = [n, n + 7, -1, -(1 << 40), 1 << 40]
        for i in range(1, T):
            if rng.random() < (0.3 if kind == 3 else 0.05):
                row[i] = bad[int(rng.integers(0, len(bad)))]
        out.append(row)
    return out


def case(ft, n, B, T, kind, max_len):
    rng = np.random.default_rng(n * 7 + B * 131 + T * 17 + len(kind) + max_len)
    hists, prompts, prm = P.rows_and_params(B, n, rng)
    if max_len < 256:  # a full slot: sequence 5 (200 tokens) is cut to max_len
        hists = [h[:max_len] for h in hists]
        prompts = [min(p, len(h)) for p, h in zip(prompts, hists)]
    tokens = make_drafts(hists, n, T, rng)
    parents = make_parents(kind, B, T, rng)
    x = P.make_logits(B * T, n, ft, rng)
    return hists, prompts, prm, tokens, parents, x


def run_device(ops, hists, prompts, prm, tokens, parents, x, ft, max_len, vocab, id_offset=0):
    h = ops.TokenHistory(len(hists), max_len, vocab)
    for b, (ids, p) in enumerate(zip(hists, prompts)):
        h.load(b, ids, p)
    pen = device_params(ops, prm)
    y = upload(x, ft)
    tk = torch.tensor(tokens, dtype=torch.int64, device="cuda")
    par = None if parents is None else torch.tensor(parents, dtype=torch.int32, device="cuda")
    snap = h.snapshot()
    ops.penalize_tokens(y[:, :x.shape[1]], h, pen, tk, par, id_offset=id_offset)
    torch.cuda.synchronize()
    assert all(torch.equal(a, b) for a, b in zip(snap, h.snapshot())), "the history was written"
    assert bool((y.view(torch.int16)[:, x.shape[1]:] == SENTINEL).all()), "padding columns written"
    return y, h, pen


SHAPES = [(1, 16, "deepest_last"), (8, 5, "random_tree"), (65, 2, "none"), (8, 8, "topk"), (3, 16, "malformed"),
          (8, 4, "star"), (8, 16, "none"), (8, 6, "chain")]


@pytest.mark.parametrize("ft", ["bf16", "fp16"])
@pytest.mark.parametrize("n", [1, 7, 4097, 152064])
@pytest.mark.parametrize("B,T,kind", SHAPES)
def test_matches_restatement(ops, ft, n, B, T, kind):
    max_len = {0: 256, 1: 204, 2: 200}[(B + T) % 3]
    hists, prompts, prm, tokens, parents, x = case(ft, n, B, T, kind, max_len)
    y, _, _ = run_device(ops, hists, prompts, prm, tokens, parents, x, ft, max_len, n)
    want, alt = PT.penalize_tokens(x, hists, prompts, tokens, parents, prm, ft, max_len, n)
    got = y[:, :n].double().cpu().numpy()
    ok = P.same(got, want) | P.same(got, alt)
    bad = np.argwhere(~ok)
    assert bad.size == 0, [(int(r), int(c), got[r, c], want[r, c], x[r, c]) for r, c in bad[:8]]


@pytest.mark.parametrize("ft", ["bf16", "fp16"])
@pytest.mark.parametrize("n", [4097, 152064])
@pytest.mark.parametrize("B,T,kind", [(8, 16, "random_tree"), (65, 3, "none"), (3, 16, "malformed"), (8, 8, "topk")])
def test_equals_penalize_on_loaded_virtual_histories(ops, ft, n, B, T, kind):
    """device against device: every V(b, t) loaded into its own slot, b2_penalize on row b*T + t: identical bits"""
    max_len = 204
    hists, prompts, prm, tokens, parents, x = case(ft, n, B, T, kind, max_len)
    y, _, _ = run_device(ops, hists, prompts, prm, tokens, parents, x, ft, max_len, n)
    virt = PT.virtual_rows(hists, prompts, tokens, parents, max_len, n)
    hv = ops.TokenHistory(B * T, max_len, n)
    for r, (V, p) in enumerate(virt):
        load_raw(ops, hv, r, V, p)
    assert hv.len.cpu().tolist() == [len(V) for V, _ in virt]
    per_row = {k: [v for v in prm[k] for _ in range(T)] for k in prm}
    z = upload(x, ft)
    ops.penalize(z[:, :n], hv, device_params(ops, per_row))
    assert torch.equal(y.view(torch.int16), z.view(torch.int16))


@pytest.mark.parametrize("ft", ["bf16", "fp16"])
def test_q_len_one_equals_penalize(ops, ft):
    n, B = 4097, 65
    hists, prompts, prm, tokens, _, x = case(ft, n, B, 1, "none", 256)
    y, h, pen = run_device(ops, hists, prompts, prm, tokens, None, x, ft, 256, n)
    z = upload(x, ft)
    ops.penalize(z[:, :n], h, pen)
    assert torch.equal(y.view(torch.int16), z.view(torch.int16))


@pytest.mark.parametrize("ft", ["bf16", "fp16"])
def test_neutral_parameters_leave_the_rows_bit_identical(ops, ft):
    n, B, T = 4097, 16, 8
    hists, prompts, _, tokens, parents, x = case(ft, n, B, T, "random_tree", 256)
    y, _, _ = run_device(ops, hists, prompts, P.neutral(B), tokens, parents, x, ft, 256, n)
    assert torch.equal(y.view(torch.int16), upload(x, ft).view(torch.int16))


@pytest.mark.parametrize("ft", ["bf16", "fp16"])
def test_vocab_shards_equal_the_whole_row(ops, ft):
    n, B, T = 152064, 9, 6
    hists, prompts, prm, tokens, parents, x = case(ft, n, B, T, "random_tree", 204)
    whole, h, pen = run_device(ops, hists, prompts, prm, tokens, parents, x, ft, 204, n)
    tk = torch.tensor(tokens, dtype=torch.int64, device="cuda")
    par = torch.tensor(parents, dtype=torch.int32, device="cuda")
    for tp in (2, 4, 8):
        w = n // tp
        parts = []
        for k in range(tp):
            part = upload(x[:, k * w:(k + 1) * w], ft)
            ops.penalize_tokens(part[:, :w], h, pen, tk, par, id_offset=k * w)
            assert bool((part.view(torch.int16)[:, w:] == SENTINEL).all())
            parts.append(part[:, :w])
        assert torch.equal(torch.cat(parts, 1).view(torch.int16), whole[:, :n].view(torch.int16)), tp


def test_graph_replay_equals_eager(ops):
    n, B, T = 152064, 8, 8
    rng = np.random.default_rng(21)
    hists, prompts, prm, _, _, _ = case("bf16", n, B, T, "none", 256)
    h = ops.TokenHistory(B, 256, n)
    for b, (ids, p) in enumerate(zip(hists, prompts)):
        h.load(b, ids, p)
    pen = device_params(ops, prm)
    feeds = [(P.make_logits(B * T, n, "bf16", rng), make_drafts(hists, n, T, rng), [SS.TREES["random_tree"](rng, T)
                                                                                   for _ in range(B)]) for _ in range(6)]
    lg = torch.empty(B * T, n, dtype=torch.bfloat16, device="cuda")
    tk = torch.zeros(B, T, dtype=torch.int64, device="cuda")
    par = torch.zeros(B, T, dtype=torch.int32, device="cuda")

    def feed(i):
        x, tokens, parents = feeds[i]
        lg.copy_(torch.from_numpy(x).to(torch.bfloat16))
        tk.copy_(torch.tensor(tokens))
        par.copy_(torch.tensor(parents))

    eager = []
    for i in range(len(feeds)):
        feed(i)
        ops.penalize_tokens(lg, h, pen, tk, par)
        eager.append(lg.clone())
    feed(0)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        ops.penalize_tokens(lg, h, pen, tk, par)
    for i in range(len(feeds)):
        feed(i)
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(lg.view(torch.int16), eager[i].view(torch.int16)), i


# ------------------------------------------------------------------------------------------------------------- streams
def _u64(a):
    return torch.from_numpy(np.asarray(a, np.uint64).view(np.int64).copy()).cuda()


def _np_u64(t):
    return t.cpu().numpy().view(np.uint64)


def _sampling(B, rng):
    """per-sequence (t, k, p, seeds, offsets), a greedy sequence included"""
    t = np.array([[0.7, 1.0, 0.0, 1.3][b % 4] for b in range(B)], np.float32)
    k = np.array([[0, 50, 1, 7][b % 4] for b in range(B)], np.int32)
    p = np.array([[1.0, 0.9, 0.5, 0.95][b % 4] for b in range(B)], np.float32)
    seeds = rng.integers(0, 2 ** 63, B, dtype=np.uint64) * np.uint64(2) + np.uint64(1)
    offs = rng.integers(0, 2 ** 63, B, dtype=np.uint64)
    return t, k, p, seeds, offs


PROMPTS = [[1, 2, 9, 1, 7, 2], [3, 8, 3, 8, 3, 8], [5, 6, 7, 4, 5, 6], [11, 9, 13, 9, 11, 12]]
PROMPT_LENS = [6, 3, 0, 4]  # the rest of each prompt counts as generated


def _penalties(oracle):
    """mixed per-sequence penalties; eos = the unpenalised first choice, banned by min_length for the first steps"""
    eos = [int(SR.order(oracle.row(p))[0]) for p in PROMPTS]
    return dict(repetition=[1.3, 1.0, 1.05, 0.8], presence=[0.5, 0.0, -0.5, 1.0], frequency=[0.0, 0.8, 0.3, -0.25],
                no_repeat_ngram=[0, 2, 3, 1], min_length=[0, 9, 10, 12], eos_id=[-1, eos[1], eos[2], eos[3]],
                suppress=[1, 0, 1, 0])


def _history(ops, vocab, max_len):
    h = ops.TokenHistory(len(PROMPTS), max_len, vocab)
    for b, p in enumerate(PROMPTS):
        h.load(b, p, PROMPT_LENS[b])
    return h


def _single_stream(ops, oracle, pen, smp, steps, greedy, max_len):
    """penalize, sample (or argmax), append: one token per step; the history after every step"""
    B = len(PROMPTS)
    h = _history(ops, oracle.vocab, max_len)
    ctx = [list(p) for p in PROMPTS]
    dev = [torch.from_numpy(a).cuda() for a in smp[:3]] + [_u64(smp[3])]
    off = _u64(smp[4])
    snaps = [h.snapshot()]
    for _ in range(steps):
        lg = G.to_ft(np.stack([oracle.row(c) for c in ctx]), oracle.dt).cuda()
        ops.penalize(lg, h, pen)
        ids = ops.argmax(lg) if greedy else ops.sample(lg, *dev, off)
        h.append(ids)
        snaps.append(h.snapshot())
        for b, v in enumerate(ids.cpu().tolist()):
            ctx[b].append(v)
    return [c[len(p):] for c, p in zip(ctx, PROMPTS)], snaps


def _spec_stream(ops, oracle, pen, smp, L, T, tree, drafter, truths, greedy, max_len, seed):
    """drafts, penalize_tokens, sample_tokens (or argmax), accept, append_tokens, until every sequence has L tokens"""
    B = len(PROMPTS)
    rng = np.random.default_rng(seed)
    h = _history(ops, oracle.vocab, max_len)
    ctx = [list(p) for p in PROMPTS]
    out = [[] for _ in range(B)]
    dev = [torch.from_numpy(a).cuda() for a in smp[:3]] + [_u64(smp[3])]
    off = _u64(smp[4])
    acc, nxt = torch.zeros(B, dtype=torch.int32, device="cuda"), torch.zeros(B, dtype=torch.int64, device="cuda")
    old, new = torch.zeros(B, dtype=torch.int32, device="cuda"), torch.zeros(B, dtype=torch.int32, device="cuda")
    path = torch.zeros(B, T, dtype=torch.int32, device="cuda")
    tk = torch.zeros(B, T, dtype=torch.int64, device="cuda")
    tk[:, 0] = torch.tensor([p[-1] for p in PROMPTS])
    dor = SS.Oracle(oracle.vocab, oracle.seed, oracle.dt, perturb=0.7) if drafter == "sampled" else None
    while min(len(o) for o in out) < L:
        if drafter == "ngram":
            par = None if tree == "chain" else torch.zeros(B, T, dtype=torch.int32, device="cuda")
            ops.ngram_draft(h, tk, par, 1, 4, 1 if par is None else min(3, T - 1))
            tokens = tk.cpu().numpy()
            pars = [SS.TREES["chain"](rng, T)] * B if par is None else par.cpu().tolist()
        else:
            pars = [SS.TREES[tree](rng, T) for _ in range(B)]
            tokens = np.stack([SS.draft(drafter, rng, oracle, ctx[b], pars[b], truths[b][len(out[b]):], dor) for b in range(B)])
            tk.copy_(torch.from_numpy(tokens))
            par = None if tree == "chain" else torch.tensor(pars, dtype=torch.int32, device="cuda")
        lg = G.to_ft(np.stack([oracle.row(c) for b in range(B) for c in SS.contexts(ctx[b], tokens[b], pars[b])]),
                     oracle.dt).cuda()
        ops.penalize_tokens(lg, h, pen, tk, par)
        pred = (ops.argmax(lg) if greedy else ops.sample_tokens(lg, T, *dev, off, parents=par)).view(B, T)
        ops._spec_accept(acc, nxt, old, new, tk, pred, path if par is not None else None, par, None if greedy else off)
        h.append_tokens(pred, acc, path if par is not None else None)
        pr, n, pa = pred.cpu().numpy(), acc.cpu().numpy(), path.cpu().numpy()
        for b in range(B):
            emitted = [int(pr[b, pa[b, i] if par is not None else i]) for i in range(n[b])]
            out[b] += emitted
            ctx[b] += emitted
    return out, _np_u64(off), h


def _same_slot(snap, h, b):
    return all(torch.equal(s[b], getattr(h, k)[b]) for s, k in zip(snap, h._FIELDS))


@pytest.mark.parametrize("vocab", [4096, 152064])
@pytest.mark.parametrize("greedy", [True, False])
def test_stream_equality_with_penalties(ops, vocab, greedy):
    """the penalised speculative loop emits the penalised single-token stream, for every drafter (the four host drafters
    and b2_ngram_draft), chains and trees, ends at the same offsets and leaves the same history arrays"""
    oracle = SS.Oracle(vocab, seed=vocab + 3)
    prm = _penalties(oracle)
    pen = device_params(ops, prm)
    smp = _sampling(len(PROMPTS), np.random.default_rng(vocab + greedy))
    L = 12
    Ts = [2, 5, 16] if vocab == 4096 else [8]
    big = 512
    truths, snaps = _single_stream(ops, oracle, pen, smp, L * max(Ts), greedy, big)
    for b in (1, 2, 3):  # eos, the unpenalised first choice, is banned until min_length
        assert prm["eos_id"][b] not in truths[b][:prm["min_length"][b] - len(PROMPTS[b])], b
    for T in Ts:
        # at T = 16 the slots fill mid-stream (max_len 30), in both loops alike
        max_len = 30 if T == 16 else big
        ref, ref_snaps = (truths, snaps) if max_len == big else _single_stream(ops, oracle, pen, smp, L * T, greedy, max_len)
        runs = [(tree, d) for tree in SS.TREES for d in SS.DRAFTERS] + [("chain", "ngram"), ("tree", "ngram")]
        for tree, drafter in runs:
            out, off, h = _spec_stream(ops, oracle, pen, smp, L, T, tree, drafter, ref, greedy, max_len, seed=T)
            for b in range(len(PROMPTS)):
                k = len(out[b])
                assert out[b] == ref[b][:k], (T, tree, drafter, b)
                if not greedy:
                    assert int(off[b]) == (int(smp[4][b]) + k) % 2 ** 64, (T, tree, drafter, b)
                assert _same_slot(ref_snaps[k], h, b), (T, tree, drafter, b)


def test_captured_speculative_tail_equals_eager(ops):
    """b2_ngram_draft, penalize_tokens, sample_tokens, the sampled accept and append_tokens captured in one graph and
    replayed 8 times, the rows rewritten between replays, equal 8 eager steps: every output and the history"""
    vocab, B, T = 152064, 4, 8
    rng = np.random.default_rng(31)
    oracle = SS.Oracle(vocab, seed=5)
    pen = device_params(ops, _penalties(oracle))
    smp = _sampling(B, rng)
    dev = [torch.from_numpy(a).cuda() for a in smp[:3]] + [_u64(smp[3])]
    h = _history(ops, vocab, 256)
    pool = rng.integers(0, vocab, 6)
    rows = []
    for _ in range(8):  # peaked at ids of a small pool, so the history repeats and the drafter finds matches
        x = rng.standard_normal((B * T, vocab))
        x[np.arange(B * T), pool[rng.integers(0, 6, B * T)]] += 12.0
        rows.append(G.to_ft(x, torch.bfloat16).cuda())
    st = dict(lg=torch.empty_like(rows[0]), pred=torch.zeros(B * T, dtype=torch.int64, device="cuda"),
              tk=torch.zeros(B, T, dtype=torch.int64, device="cuda"), par=torch.zeros(B, T, dtype=torch.int32, device="cuda"),
              acc=torch.zeros(B, dtype=torch.int32, device="cuda"), nxt=torch.zeros(B, dtype=torch.int64, device="cuda"),
              old=torch.zeros(B, dtype=torch.int32, device="cuda"), new=torch.zeros(B, dtype=torch.int32, device="cuda"),
              path=torch.zeros(B, T, dtype=torch.int32, device="cuda"), off=_u64(smp[4]))

    def step():
        ops.ngram_draft(h, st["tk"], st["par"], 1, 4, 3)
        ops.penalize_tokens(st["lg"], h, pen, st["tk"], st["par"])
        ops.sample_tokens(st["lg"], T, *dev, st["off"], parents=st["par"], out=st["pred"])
        pv = st["pred"].view(B, T)
        ops._spec_accept(st["acc"], st["nxt"], st["old"], st["new"], st["tk"], pv, st["path"], st["par"], st["off"])
        h.append_tokens(pv, st["acc"], st["path"])

    start = h.snapshot()

    def reset():
        h.restore(start)
        for k in ("tk", "par", "acc", "old", "new", "path", "pred"):
            st[k].zero_()
        st["tk"][:, 0] = torch.tensor([p[-1] for p in PROMPTS])
        st["off"].copy_(_u64(smp[4]))

    def run(replay):
        reset()
        outs = []
        for i in range(8):
            st["lg"].copy_(rows[i])
            replay() if replay else step()
            torch.cuda.synchronize()
            outs.append([st[k].clone() for k in ("lg", "pred", "acc", "path", "par", "tk", "off")] + h.snapshot())
        return outs

    eager = run(None)
    reset()
    st["lg"].copy_(rows[0])
    step()  # warm-up, then capture
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        step()
    replayed = run(g.replay)
    for i in range(8):
        for j, (a, b) in enumerate(zip(eager[i], replayed[i])):
            assert torch.equal(a, b), (i, j)
