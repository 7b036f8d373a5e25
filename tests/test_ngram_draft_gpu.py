"""GPU: b2_ngram_draft equals the restatement (tests/ngram_ref.py) bit for bit, and b2_history_append_tokens equals
successive b2_history_append calls in every array of the history."""
import ctypes as C

import numpy as np
import pytest
import torch

import ngram_ref as N

pytestmark = pytest.mark.gpu

SENT = -77  # guard value around every output


def _histories(rng, T):
    """ragged histories of every kind: (name, token list)"""
    out = [("empty", []), ("one", [5]), ("two", [5, 5]), ("three", [3, 4, 3])]
    for L in (17, 4097):
        out.append(("rand%d" % L, rng.integers(0, 6, L).tolist()))       # many short matches
        out.append(("wide%d" % L, rng.integers(0, 50000, L).tolist()))   # few matches
    for p in range(1, T + 2):                                            # periodic: the early exit
        seg = rng.integers(0, 1000, p).tolist()
        out.append(("period%d" % p, (rng.integers(0, 1000, 5).tolist() + seg * (60 // p + 2))[:60 + p]))
    eq = []
    for _ in range(20):                                                  # many equal-length matches, distinct continuations
        eq += [1, 2, 3, int(rng.integers(10, 40))]
    out.append(("equal", eq + [1, 2, 3]))
    neg = rng.integers(0, 4, 300).tolist()                               # -1 entries
    for i in range(0, 300, 7):
        neg[i] = -1
    out.append(("minus1", neg + [-1]))
    return out


def _long_histories(rng):
    """131072 tokens: one needle at the very start, a random one, a periodic one"""
    L = 131072
    needle = (np.arange(L) + 1000).tolist()
    needle[:3] = [7, 8, 9]
    needle[-3:] = [7, 8, 9]
    seg = rng.integers(0, 1000, 5).tolist()
    return [("needle", needle), ("rand128k", rng.integers(0, 150000, L).tolist()), ("period128k", (seg * (L // 5 + 1))[:L])]


def _load(hists, max_len, device="cuda"):
    """a TokenHistory whose tokens / len are the lists (the drafter reads nothing else)"""
    from b200spark import ops
    h = ops.TokenHistory(len(hists), max_len, 200000, device)
    tok = torch.full((len(hists), max_len), -1, dtype=torch.int32)
    for b, S in enumerate(hists):
        tok[b, :len(S)] = torch.tensor(S, dtype=torch.int32)
    h.tokens.copy_(tok)
    h.len.copy_(torch.tensor([len(S) for S in hists], dtype=torch.int32))
    return h


def _outputs(B, T, tree, tok0):
    """tokens / parents / n_draft views inside guard-filled buffers"""
    tb = torch.full((B * T + 8,), SENT, dtype=torch.int64, device="cuda")
    tokens = tb[:B * T].view(B, T)
    tokens[:, 0] = tok0
    pb = torch.full((B * T + 8,), SENT, dtype=torch.int32, device="cuda") if tree else None
    nb = torch.full((B + 8,), SENT, dtype=torch.int32, device="cuda")
    return tb, tokens, pb, (pb[:B * T].view(B, T) if tree else None), nb, nb[:B]


def _check(hists, cands, tok0, T, width, tree, tb, pb, nb):
    B = len(hists)
    want = [N.draft_from(S, c[:width], int(t), T, tree) for S, c, t in zip(hists, cands, tok0)]
    got_t = tb[:B * T].view(B, T).tolist()
    assert tb[B * T:].eq(SENT).all() and nb[B:].eq(SENT).all()
    for b in range(B):
        assert got_t[b] == want[b][0], (b, T, width, tree, got_t[b], want[b][0])
        assert int(nb[b]) == want[b][2], (b, T, width, tree)
    if tree:
        assert pb[B * T:].eq(SENT).all()
        got_p = pb[:B * T].view(B, T).tolist()
        for b in range(B):
            assert got_p[b] == want[b][1], (b, T, width, got_p[b], want[b][1])


@pytest.mark.parametrize("ngram", [(1, 1), (1, 4), (3, 3), (2, 16)])
def test_draft_matches_restatement(ngram):
    from b200spark import ops
    n_min, n_max = ngram
    rng = np.random.default_rng(n_min * 31 + n_max)
    named = _histories(rng, 16)
    named += [named[i % len(named)] for i in range(65 - len(named))]     # 65 rows, ragged
    hists = [S for _, S in named]
    h = _load(hists, 4200)
    tok0 = torch.tensor([S[-1] if S else 11 for S in hists], dtype=torch.int64, device="cuda")
    cands = [N.candidates(S, n_min, n_max, 15) for S in hists]
    for B in (65, 64, 1):
        for T in range(2, 17):
            for width in range(1, min(8, T - 1) + 1):
                for tree in ((False, True) if width == 1 else (True,)):
                    tb, tokens, pb, parents, nb, n_draft = _outputs(B, T, tree, tok0[:B])
                    ops.ngram_draft(h.view(B), tokens, parents, n_min, n_max, width, n_draft=n_draft)
                    torch.cuda.synchronize()
                    _check(hists[:B], cands[:B], tok0[:B].tolist(), T, width, tree, tb, pb, nb)
            if B != 65:
                break  # the other batches at T = 2 only


def test_long_histories():
    from b200spark import ops
    rng = np.random.default_rng(5)
    named = _long_histories(rng)
    hists = [S for _, S in named]
    h = _load(hists, 131072)
    tok0 = torch.tensor([S[-1] for S in hists], dtype=torch.int64, device="cuda")
    for n_min, n_max in ((1, 1), (1, 4), (3, 3), (2, 16)):
        cands = [N.candidates(S, n_min, n_max, 15) for S in hists]
        if n_max >= 3:
            assert cands[0] == [2], cands[0]  # the needle: the earliest possible match
        for T, width, tree in ((2, 1, False), (8, 1, False), (8, 4, True), (16, 8, True), (16, 15, True)):
            tb, tokens, pb, parents, nb, n_draft = _outputs(3, T, tree, tok0)
            ops.ngram_draft(h, tokens, parents, n_min, n_max, width, n_draft=n_draft)
            torch.cuda.synchronize()
            _check(hists, cands, tok0.tolist(), T, width, tree, tb, pb, nb)


def test_graph_replay_equals_eager():
    from b200spark import ops
    rng = np.random.default_rng(9)
    hists = [S for _, S in _histories(rng, 8)]
    h = _load(hists, 4200)
    B = len(hists)
    tok0 = torch.tensor([S[-1] if S else 11 for S in hists], dtype=torch.int64, device="cuda")
    for tree, width in ((False, 1), (True, 3)):
        eager = _outputs(B, 8, tree, tok0)
        graph = _outputs(B, 8, tree, tok0)
        ops.ngram_draft(h, eager[1], eager[3], 1, 4, width, n_draft=eager[5])
        g = torch.cuda.CUDAGraph()
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            with torch.cuda.graph(g):
                ops.ngram_draft(h, graph[1], graph[3], 1, 4, width, n_draft=graph[5])
        torch.cuda.current_stream().wait_stream(s)
        g.replay()
        torch.cuda.synchronize()
        for i in (0, 2, 4):
            if eager[i] is not None:
                assert torch.equal(eager[i], graph[i]), (tree, i)


def _slot(h, b):
    """the C view of slot b alone (a one-row history at the slot's addresses)"""
    from b200spark import _lib
    return _lib.TokenHistory(h.tokens[b].data_ptr(), h.len[b:].data_ptr(), h.prompt_len[b:].data_ptr(), h.table[b].data_ptr(),
                             h.distinct[b].data_ptr(), h.n_distinct[b:].data_ptr(), h.max_len, h.vocab)


def _arrays(h):
    return [getattr(h, k).clone() for k in h._FIELDS]


@pytest.mark.parametrize("tree", [False, True])
def test_append_tokens_equals_successive_appends(tree):
    from b200spark import _lib, ops
    B, T, max_len, vocab = 9, 6, 40, 64
    rng = np.random.default_rng(4 + tree)
    a, ref = ops.TokenHistory(B, max_len, vocab), ops.TokenHistory(B, max_len, vocab)
    for b in range(B):
        n = max_len - 2 if b == 3 else int(rng.integers(0, 12))          # slot 3 fills up mid-step
        a.load(b, rng.integers(0, 8, n).tolist(), n // 2)
    ref.restore(a.snapshot())  # the load orders the distinct list by atomics: start both from the same arrays
    for step in range(4):
        pred = torch.tensor(rng.integers(0, 10, (B, T)), dtype=torch.int64, device="cuda")
        pred[0, 1] = vocab + 5                                            # an id outside the vocabulary: stored as -1
        acc = torch.tensor([(b + step) % T + 1 for b in range(B)], dtype=torch.int32, device="cuda")
        path = None
        if tree:  # a path of increasing node indices from node 0
            path = torch.zeros(B, T, dtype=torch.int32)
            for b in range(B):
                nodes = sorted(rng.choice(np.arange(1, T), T - 1, replace=False)[:int(acc[b]) - 1].tolist())
                path[b, 1:1 + len(nodes)] = torch.tensor(nodes, dtype=torch.int32)
            path = path.cuda()
        a.append_tokens(pred, acc, path)
        for b, ids in enumerate(N.emitted(pred.tolist(), acc.tolist(), None if path is None else path.tolist())):
            one = _slot(ref, b)
            for t in ids:
                _lib.check(_lib.lib.b2_history_append(C.byref(one), ops._ptr(torch.tensor([t], dtype=torch.int64,
                                                                                         device="cuda")), 1, ops._stream()))
        torch.cuda.synchronize()
        for k, x, y in zip(a._FIELDS, _arrays(a), _arrays(ref)):
            assert torch.equal(x, y), (k, step)
    assert int(a.len[3]) == max_len


def test_append_tokens_graph_replay_appends_once_per_replay():
    from b200spark import ops
    B, T = 4, 4
    a, e = ops.TokenHistory(B, 64, 100), ops.TokenHistory(B, 64, 100)
    for b in range(B):
        a.load(b, [b, b + 1])
    e.restore(a.snapshot())
    pred = torch.arange(B * T, dtype=torch.int64, device="cuda").view(B, T)
    acc = torch.tensor([1, 2, 3, 4], dtype=torch.int32, device="cuda")
    for h in (a, e):  # an eager call first: the kernel is loaded before capture
        h.append_tokens(pred, acc)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(g):
            a.append_tokens(pred, acc)
    torch.cuda.current_stream().wait_stream(s)
    for _ in range(3):
        g.replay()
        e.append_tokens(pred, acc)
    torch.cuda.synchronize()
    assert all(torch.equal(x, y) for x, y in zip(_arrays(a), _arrays(e)))
    assert a.len.tolist() == [6, 10, 14, 18]
