"""GPU: sampling under tensor parallelism (b2_sample_shard, b2_sample_shard_merge) against b2_sample on the whole rows,
bit for bit.  Both sides weigh every element with the same code at the same m and c, so no ambiguity allowance applies:
every rank's ids and offsets must equal b2_sample's on any row.

The ranks are simulated on one device: each "rank" runs the phases on its column range of one logits tensor with its own
state and its own copies of the parameters, and the records are exchanged by stacking them with torch, or by loopback
communicators (b2_allgather, every rank on its own stream)."""
import numpy as np
import pytest
import torch

import sample_ref as S
import sample_tp_ref as T

pytestmark = pytest.mark.gpu

PHASES = 6


def _ops():
    from b200spark import ops
    return ops


def _rows(B, n, dt, bounds, gen, rng):
    """[B, n] logits cycling through the row kinds: exact, N(0, 1) flat, peaked, a NaN, a +inf, all -inf, and needles: equal
    maxima on both sides of every shard boundary (a run of ties the ranks share)"""
    x = torch.randn(B, n, generator=gen, device="cuda")
    for r in range(B):
        kind = r % 7
        if kind == 0:
            x[r] = torch.from_numpy(S.exact_row(n, r % 3, 0.0 if r % 2 else 2.0, rng, dt, neg_inf=2)).cuda()
        elif kind == 2:
            x[r] = x[r] * 4
            x[r, int(rng.integers(0, n))] = 24.0
        elif kind == 3:
            x[r, int(rng.integers(0, n))] = float("nan")
        elif kind == 4:
            x[r, int(rng.integers(0, n))] = float("inf")
        elif kind == 5:
            x[r] = float("-inf")
        elif kind == 6:
            x[r] = x[r] - 8
            for b in bounds[1:-1]:
                x[r, b - 1] = x[r, b] = 3.0
            x[r, bounds[-1] - 1] = 3.0
    return x.to(dt)


def _params(B, n, gen):
    """per-row parameters cycling through every kind: t <= 0, t = inf, k = 1, k = n, k > n, tiny p, p = 1, NaN p, and a
    realistic (0.7, 50, 0.9)"""
    kinds = [(0.0, 0, 1.0), (float("inf"), 0, 1.0), (1.0, 1, 1.0), (1.0, n, 1.0), (1.0, n + 5, 0.5), (0.8, 0, 1e-6),
             (1.3, 0, 1.0), (1.0, 40, float("nan")), (0.7, 50, 0.9), (-1.0, 7, 0.3), (1.0, 0, 0.95)]
    t = torch.tensor([kinds[r % len(kinds)][0] for r in range(B)], dtype=torch.float32, device="cuda")
    k = torch.tensor([kinds[r % len(kinds)][1] for r in range(B)], dtype=torch.int32, device="cuda")
    p = torch.tensor([kinds[r % len(kinds)][2] for r in range(B)], dtype=torch.float32, device="cuda")
    seeds = torch.randint(0, 2**62, (B,), generator=gen, device="cuda", dtype=torch.int64)
    offs = torch.randint(0, 2**40, (B,), generator=gen, device="cuda", dtype=torch.int64)
    return t, k, p, seeds, offs


class Ranks:
    """P simulated ranks over the column ranges `bounds` of one logits tensor; stacking exchange into fixed buffers (so a
    graph can capture a whole protocol)"""

    def __init__(self, bounds, B, params):
        ops = _ops()
        self.bounds, self.P = bounds, len(bounds) - 1
        self.bufs = [ops.sample_tp_buffers(B, self.P) for _ in range(self.P)]
        self.params = [[t.clone() for t in params] for _ in range(self.P)]  # every rank its own device copies
        self.ids = [torch.empty(B, dtype=torch.int64, device="cuda") for _ in range(self.P)]

    def run(self, logits):
        ops = _ops()
        n_total = self.bounds[-1]
        for ph in range(PHASES):
            for q in range(self.P):
                a, e = self.bounds[q], self.bounds[q + 1]
                ops.sample_shard(ph, logits[:, a:e], a, n_total, *self.params[q], self.bufs[q]["state"],
                                 self.bufs[q]["all"][ph - 1] if ph else None, out=self.bufs[q]["rec"][ph], nranks=self.P)
            for q in range(self.P):
                for s in range(self.P):
                    self.bufs[q]["all"][ph][s].copy_(self.bufs[s]["rec"][ph].view(-1))
        for q in range(self.P):
            ops.sample_shard_merge(self.bufs[q]["all"][PHASES - 1], self.bufs[q]["state"], self.params[q][4], out=self.ids[q])
        return self.ids


def _check(logits, bounds, params):
    ops = _ops()
    ranks = Ranks(bounds, logits.shape[0], params)
    offs_ref = params[4].clone()
    want = ops.sample(logits, *params[:4], offs_ref)
    got = ranks.run(logits)
    torch.cuda.synchronize()
    for q in range(ranks.P):
        bad = (got[q] != want).nonzero().flatten().tolist()
        assert not bad, (q, bounds, bad[:8], got[q][bad[:8]].tolist(), want[bad[:8]].tolist())
        assert torch.equal(ranks.params[q][4], offs_ref), q
    return want


@pytest.mark.parametrize("P", [1, 2, 3, 4, 8])
@pytest.mark.parametrize("n_total", [4097, 151936, 152064, 262144])
@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("split", ["even", "uneven"])
def test_bit_exact_against_b2_sample(P, n_total, dt, split):
    rng = np.random.default_rng(P * 7 + n_total + (dt == torch.float16))
    gen = torch.Generator(device="cuda").manual_seed(P * 13 + n_total)
    bounds = T.even_bounds(n_total, P) if split == "even" else T.random_bounds(n_total, P, rng, one_col=P > 2)
    B = 65 if split == "even" else 16
    _check(_rows(B, n_total, dt, bounds, gen, rng), bounds, _params(B, n_total, gen))


@pytest.mark.parametrize("B", [1, 16, 64, 65])
def test_batch_sizes(B):
    rng = np.random.default_rng(B)
    gen = torch.Generator(device="cuda").manual_seed(B)
    bounds = T.random_bounds(152064, 4, rng)
    _check(_rows(B, 152064, torch.bfloat16, bounds, gen, rng), bounds, _params(B, 152064, gen))


def test_4096_consecutive_offsets_of_one_row():
    """one realistic row drawn at 4096 consecutive counters (rows of one batch), split over 4 unequal ranks"""
    gen = torch.Generator(device="cuda").manual_seed(3)
    n, B = 152064, 4096
    row = (torch.randn(n, generator=gen, device="cuda") * 3).to(torch.bfloat16)
    logits = row.expand(B, n).contiguous()
    params = (torch.full((B,), 0.9, device="cuda"), torch.full((B,), 0, dtype=torch.int32, device="cuda"),
              torch.full((B,), 0.95, device="cuda"), torch.full((B,), 1234, dtype=torch.int64, device="cuda"),
              torch.arange(B, dtype=torch.int64, device="cuda"))
    want = _check(logits, [0, 20000, 90001, 90002, n], params)
    assert want.unique().numel() > 16  # the draws do vary with the counter


def test_graph_replay_advances_offsets_and_equals_eager():
    rng = np.random.default_rng(11)
    gen = torch.Generator(device="cuda").manual_seed(11)
    n, B = 151936, 16
    bounds = T.even_bounds(n, 2)
    logits = _rows(B, n, torch.bfloat16, bounds, gen, rng)
    params = _params(B, n, gen)
    eager = Ranks(bounds, B, params)
    graphed = Ranks(bounds, B, params)
    graphed.run(logits)  # warm-up, then rewind the counters
    torch.cuda.synchronize()
    for q in range(2):
        graphed.params[q][4].copy_(params[4])
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        graphed.run(logits)
    for q in range(2):
        graphed.params[q][4].copy_(params[4])
    for it in range(3):
        want = [i.clone() for i in eager.run(logits)]
        g.replay()
        torch.cuda.synchronize()
        for q in range(2):
            assert torch.equal(graphed.ids[q], want[q]), (it, q)
            assert torch.equal(graphed.params[q][4], params[4] + it + 1), (it, q)


@pytest.mark.parametrize("P", [2, 4, 8])
def test_loopback_communicators(P):
    """records moved by b2_allgather between loopback communicators, every rank on its own stream: eagerly, then with
    per-rank captured graphs replayed concurrently"""
    ops = _ops()
    rng = np.random.default_rng(P)
    gen = torch.Generator(device="cuda").manual_seed(P)
    n, B = 152064, 8
    bounds = T.random_bounds(n, P, rng)
    logits = _rows(B, n, torch.bfloat16, bounds, gen, rng)
    params = _params(B, n, gen)
    ref_offs = params[4].clone()
    want1 = ops.sample(logits, *params[:4], ref_offs)
    want2 = ops.sample(logits, *params[:4], ref_offs)
    comms = ops.Comm.connect_local([ops.Comm(q, P, B * 3072) for q in range(P)])
    streams = [torch.cuda.Stream() for _ in range(P)]
    shards = [logits[:, bounds[q]:bounds[q + 1]] for q in range(P)]
    prm = [[t.clone() for t in params] for _ in range(P)]
    bufs = [ops.sample_tp_buffers(B, P) for _ in range(P)]
    ids = [torch.empty(B, dtype=torch.int64, device="cuda") for _ in range(P)]

    def rank(q):
        ops.sample_tp(shards[q], bounds[q], n, *prm[q], lambda rec, all_: comms[q].allgather(rec, all_), P, out=ids[q],
                      bufs=bufs[q])

    torch.cuda.synchronize()
    for q in range(P):
        with torch.cuda.stream(streams[q]):
            rank(q)
    torch.cuda.synchronize()
    for c in comms:
        c.check_error()
    for q in range(P):
        assert torch.equal(ids[q], want1), q
        assert torch.equal(prm[q][4], params[4] + 1), q
    graphs = [torch.cuda.CUDAGraph() for _ in range(P)]
    for q in range(P):  # nothing runs during capture; the peers meet at replay
        with torch.cuda.graph(graphs[q], stream=streams[q]):
            rank(q)
    for q in range(P):
        with torch.cuda.stream(streams[q]):
            graphs[q].replay()
    torch.cuda.synchronize()
    for c in comms:
        c.check_error()
    for q in range(P):
        assert torch.equal(ids[q], want2), q
        assert torch.equal(prm[q][4], params[4] + 2), q
