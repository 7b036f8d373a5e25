"""GPU: b2_penalize against its restatement (tests/penalty_ref.py) bit for bit, over vocab shards, and the token history
(b2_history_load / _append) against its definition, including graph replay."""
import numpy as np
import pytest
import torch

import penalty_ref as P

pytestmark = pytest.mark.gpu

PAD = 5  # columns n .. n + PAD - 1 of every row hold a sentinel that must survive
SENTINEL = 0x7E11


@pytest.fixture(scope="module")
def ops():
    from b200spark import ops as o
    return o


def upload(ops, x, ft):
    rows, n = x.shape
    t = torch.empty(rows, n + PAD, dtype=P.FTS[ft], device="cuda")
    t.view(torch.int16)[:, n:] = SENTINEL
    t[:, :n] = torch.from_numpy(x).to(P.FTS[ft]).cuda()
    return t


def device_history(ops, hists, prompts, max_len, vocab):
    h = ops.TokenHistory(len(hists), max_len, vocab)
    for r, (ids, p) in enumerate(zip(hists, prompts)):
        h.load(r, ids, p)
    return h


def device_params(ops, prm):
    pen = ops.Penalties(len(prm["repetition"]))
    for k in P.neutral(0):
        getattr(pen, k).copy_(torch.tensor(prm[k]))
    return pen


def check(y, x, hists, prompts, prm, ft, off=0):
    rows, n = x.shape
    tok = np.full((rows, max(1, max(len(h) for h in hists))), -1, np.int64)
    for r, h in enumerate(hists):
        tok[r, :len(h)] = h
    want, alt = P.penalize(x, tok, [len(h) for h in hists], prompts, prm, ft, off)
    got = y[:, :n].double().cpu().numpy()
    ok = P.same(got, want) | P.same(got, alt)
    bad = np.argwhere(~ok)
    assert bad.size == 0, [(int(r), int(c), got[r, c], want[r, c], x[r, c]) for r, c in bad[:8]]
    assert bool((y.view(torch.int16)[:, n:] == SENTINEL).all()), "padding columns written"
    return int(np.sum(~P.same(want, alt)))


@pytest.mark.parametrize("ft", ["bf16", "fp16"])
@pytest.mark.parametrize("n", [1, 7, 4097, 152064])
@pytest.mark.parametrize("rows", [1, 64, 65])
def test_matches_restatement(ops, ft, n, rows):
    hists, prompts, prm, x = P.case(ft, n, rows)
    hist = device_history(ops, hists, prompts, 256, n)
    pen = device_params(ops, prm)
    y = upload(ops, x, ft)
    ops.penalize(y[:, :n], hist, pen)
    check(y, x, hists, prompts, prm, ft)


@pytest.mark.parametrize("ft", ["bf16", "fp16"])
def test_neutral_parameters_leave_the_row_bit_identical(ops, ft):
    rng = np.random.default_rng(3)
    rows, n = 16, 4097
    hists, prompts, _ = P.rows_and_params(rows, n, rng)
    x = P.make_logits(rows, n, ft, rng)
    hist = device_history(ops, hists, prompts, 256, n)
    y = upload(ops, x, ft)
    before = y.clone()
    ops.penalize(y[:, :n], hist, ops.Penalties(rows))
    assert torch.equal(y.view(torch.int16), before.view(torch.int16))


@pytest.mark.parametrize("ft", ["bf16", "fp16"])
def test_division_over_every_positive_value(ops, ft):
    """x / R for the positive finite FT x (each id of the row occurs once, in the prompt), six values of R: bit for bit
    wherever the exact quotient is not within the restatement's window of a rounding boundary, one neighbour there"""
    dt = P.FTS[ft]
    # bf16 from 2^-125 up: every quotient by R <= 2 stays a normal number (fp16 values are all normal in fp32)
    xs = torch.arange(1 if ft == "fp16" else 0x0100, 0x7C00 if ft == "fp16" else 0x7F80, dtype=torch.int32).to(torch.int16)
    xs = xs.view(dt).double().numpy()
    n, rows = xs.size, 6
    hist = ops.TokenHistory(rows, n, n)
    for r in range(rows):
        hist.load(r, np.arange(n), n)
    prm = dict(P.neutral(rows), repetition=[1.05, 2.0, 0.5, 1.3, 0.7, 1.999])
    y = upload(ops, np.tile(xs, (rows, 1)), ft)
    ops.penalize(y[:, :n], hist, device_params(ops, prm))
    got = y[:, :n].double().cpu().numpy()
    amb = 0
    for r in range(rows):
        q = xs / P.rn(prm["repetition"][r], ft)[()]
        w = P.rn(q, ft)
        lo, hi = P.rn(q * (1 - P.DIV_REL), ft), P.rn(q * (1 + P.DIV_REL), ft)
        window = (lo != w) | (hi != w)
        ok = (got[r] == w) | (window & ((got[r] == lo) | (got[r] == hi)))
        assert ok.all(), [(xs[i], got[r, i], w[i]) for i in np.argwhere(~ok)[:8, 0]]
        amb += int(window.sum())
    assert amb <= n * rows // 100, amb


@pytest.mark.parametrize("ft", ["bf16", "fp16"])
def test_vocab_shards_equal_the_whole_row(ops, ft):
    rng = np.random.default_rng(5)
    rows, n = 65, 152064
    hists, prompts, prm = P.rows_and_params(rows, n, rng)
    x = P.make_logits(rows, n, ft, rng)
    hist = device_history(ops, hists, prompts, 256, n)
    pen = device_params(ops, prm)
    whole = upload(ops, x, ft)
    ops.penalize(whole[:, :n], hist, pen)
    for tp in (2, 4, 8):
        parts = []
        w = n // tp
        for k in range(tp):
            part = upload(ops, x[:, k * w:(k + 1) * w], ft)
            ops.penalize(part[:, :w], hist, pen, id_offset=k * w)
            assert bool((part.view(torch.int16)[:, w:] == SENTINEL).all())
            parts.append(part[:, :w])
        assert torch.equal(torch.cat(parts, 1).view(torch.int16), whole[:, :n].view(torch.int16)), tp


def history_state(h):
    nd = h.n_distinct.cpu().tolist()
    L = h.len.cpu().tolist()
    tok = h.tokens.cpu().numpy()
    return (L, h.prompt_len.cpu().tolist(), [tok[r, :L[r]].tolist() for r in range(h.rows)], h.table.cpu().numpy(),
            [sorted(h.distinct[r, :nd[r]].cpu().tolist()) for r in range(h.rows)])


def same_state(a, b):
    return a[0] == b[0] and a[1] == b[1] and a[2] == b[2] and np.array_equal(a[3], b[3]) and a[4] == b[4]


def test_history_appends_equal_one_load(ops):
    rng = np.random.default_rng(7)
    rows, max_len, vocab, T = 5, 300, 1000, 120
    seqs = [rng.integers(0, 50 if r % 2 else vocab, 160) for r in range(rows)]
    a, b = ops.TokenHistory(rows, max_len, vocab), ops.TokenHistory(rows, max_len, vocab)
    ref = P.History(rows, max_len, vocab)
    for r in range(rows):
        a.load(r, seqs[r][:40])
        b.load(r, seqs[r][:40 + T], 40)
        ref.load(r, seqs[r][:40 + T], 40)
    for j in range(40, 40 + T):
        a.append(torch.tensor([s[j] for s in seqs], dtype=torch.int64, device="cuda"))
    sa, sb = history_state(a), history_state(b)
    assert same_state(sa, sb)
    assert sa[2] == ref.tokens and sa[1] == ref.prompt
    for r in range(rows):
        e = ref.table(r)
        assert sorted(e) == sa[4][r] and all(sa[3][r, t] == v for t, v in e.items()) and int(sa[3][r].astype(bool).sum()) == len(e)


def test_reload_leaves_no_trace_and_full_slots_stay(ops):
    rows, max_len, vocab = 3, 64, 500
    rng = np.random.default_rng(9)
    h, fresh = ops.TokenHistory(rows, max_len, vocab), ops.TokenHistory(rows, max_len, vocab)
    for r in range(rows):
        h.load(r, rng.integers(0, vocab, 60), 30)
    h.append(torch.tensor([1, 2, 3], dtype=torch.int64, device="cuda"))
    new = [rng.integers(0, vocab, k) for k in (5, 0, 64)]
    for r in range(rows):
        h.load(r, new[r], len(new[r]) // 2)
        fresh.load(r, new[r], len(new[r]) // 2)
    assert same_state(history_state(h), history_state(fresh))
    h.reset(0)
    fresh.reset(0)
    # slot 2 is full: an append leaves it; an id outside the vocabulary is stored as -1 and counted nowhere
    h.append(torch.tensor([vocab + 3, -2, 7], dtype=torch.int64, device="cuda"))
    s = history_state(h)
    assert s[0] == [1, 1, 64] and s[2][0] == [-1] and s[2][1] == [-1] and s[4][0] == [] and s[4][1] == []
    assert s[2][2] == new[2].tolist() and np.array_equal(s[3][2], history_state(fresh)[3][2])


def test_graph_replay_appends_once_per_row(ops):
    rows, max_len, vocab = 4, 64, 100
    h = ops.TokenHistory(rows, max_len, vocab)
    ref = P.History(rows, max_len, vocab)
    for r in range(rows):
        h.load(r, [r, r + 1], 1)
        ref.load(r, [r, r + 1], 1)
    ids = torch.zeros(rows, dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        h.append(ids)
    torch.cuda.synchronize()
    assert history_state(h)[0] == [2] * rows  # capturing ran nothing
    for k in range(5):
        v = [(3 * k + r) % 7 for r in range(rows)]
        ids.copy_(torch.tensor(v))
        g.replay()
        ref.append(v)
    torch.cuda.synchronize()
    st = history_state(h)
    assert st[0] == [7] * rows and st[2] == ref.tokens
    for r in range(rows):
        e = ref.table(r)
        assert sorted(e) == st[4][r] and all(st[3][r, t] == v for t, v in e.items())
