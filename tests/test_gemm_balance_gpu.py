"""GPU: the wgmma GEMM's schedule (tests/tc_schedule.py) on exact-arithmetic inputs (tests/gemm_exact.py) and on random ones.

With more n-groups than SMs, each n-group left over after the whole rounds is cut in two k-ordered halves on two CTAs, the
second starting from the first's accumulators: the results must be bit-identical to B2_GEMM_TC_MAX_SPLIT=1 (every n-group
whole on one CTA) on ANY inputs, at batches 17 / 32 / 64 and over two launches (80), over a second launch and CUDA-graph
replays (the arrival counters re-arm themselves).  The k-sliced plans of fewer n-groups are checked on exact inputs against
the unsliced plan and the restatement.  The handle's workspace size is the restated plan's."""
import numpy as np
import pytest
import torch

import gemm_exact as X
import tc_schedule as TS
from test_gemm_exact_gpu import GUARD, Framed, _acts, _handle

pytestmark = pytest.mark.gpu

CASES = [
    # o_proj shape: 28 n-groups x 4 slices
    X.GpuCase("bal-o-m64", X.Case(4, 3584, 3584), 64, "tc", res=True),
    # down_proj shape: 296 k-tiles per n-group
    X.GpuCase("bal-down-m32", X.Case(4, 18944, 3584), 32, "tc", res=True, J=1),
    # 148 n-groups: one round of whole n-groups, then 16 n-groups in two halves (MULTI)
    X.GpuCase("bal-multi-m64", X.Case(4, 3584, 18944), 64, "tc", act=X.ACT_SIGMOID),
    # the gate+up pair: two rounds, then 32 pair n-groups in two halves; SwiGLU epilogue by the tail
    X.GpuCase("bal-pair-m64", X.Case(4, 3584, 18944, pair=True), 64, "tc", J=2),
    X.GpuCase("bal-pair-m80", X.Case(4, 3584, 18944, pair=True), 80, "tc", J=2),
    # int8 weights (two k-tiles per stage) in halves
    X.GpuCase("bal-w8-multi-m40", X.Case(8, 1024, 18944), 40, "tc", bias=True, J=1),
    # two launches of one call, a small K and N not a multiple of 128 (k-slices)
    X.GpuCase("bal-tail80", X.Case(4, 1024, 1290), 80, "tc", res=True, bias=True),
]


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _plan(case, max_split=TS.MAX_SPLIT):
    return TS.plan(case.NG, case.KT, _sms(), max_split)


def _graph(fn):
    g, s = torch.cuda.CUDAGraph(), torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s), torch.cuda.graph(g, stream=s):
        fn()
    torch.cuda.current_stream().wait_stream(s)
    return g


@pytest.mark.parametrize("gc", CASES, ids=lambda g: g.id)
def test_balanced_matches_unshared(gc, monkeypatch):
    from b200spark import ops
    c = gc.case
    inp = X.dyadic_inputs(gc)
    X.case_precondition(gc, inp)
    y, E = X.restate(gc, inp)
    A = _acts(inp["A"], torch.bfloat16, 0)
    res = Framed(gc.M, c.N, torch.bfloat16, GUARD).fill(torch.from_numpy(inp["res"]).to(torch.bfloat16)).view \
        if inp["res"] is not None else None
    pl = _plan(c)
    assert pl.S > 1 or pl.h > 0, pl               # some n-groups are split
    outs = []
    for ms in (None, "1"):
        if ms:
            monkeypatch.setenv("B2_GEMM_TC_MAX_SPLIT", ms)
        op = _handle(gc, inp)
        assert op.workspace_bytes(gc.M) == _plan(c, int(ms or TS.MAX_SPLIT)).workspace_bytes(), gc.id
        fr = Framed(gc.M, c.N, torch.bfloat16, GUARD)
        ws = ops.Workspace()
        run = lambda out: op(A, ws, out=out, act=gc.act, alpha=gc.alpha, residual=res)
        run(fr.view)
        first = fr.view.clone()
        run(fr.view)
        fr2 = Framed(gc.M, c.N, torch.bfloat16, GUARD)
        g = _graph(lambda: run(fr2.view))
        for _ in range(3):
            g.replay()
        torch.cuda.synchronize()
        assert torch.equal(fr.view, first) and torch.equal(fr2.view, first), f"{gc.id}: repeat / replay differs"
        assert fr.guards_intact() and fr2.guards_intact()
        outs.append(first)
        monkeypatch.delenv("B2_GEMM_TC_MAX_SPLIT", raising=False)
    assert torch.equal(outs[0], outs[1]), f"{gc.id}: balanced != unshared"
    bad, _ = X.check(outs[0].double().cpu().numpy(), y, E, c.ft)
    assert not bad.any(), f"{gc.id}: {int(bad.sum())} elements off the restatement"


@pytest.mark.parametrize("M", [17, 32, 64, 80])
def test_handoff_outputs_balanced(M, monkeypatch):
    """xg_out and sumsq_out are written by the last k-slice of each n-group to arrive: bit-identical to the unsliced plan,
    over a graph replay too."""
    from b200spark import ops
    gc = X.GpuCase("bal-handoff", X.Case(4, 1024, 1280), M, "tc", res=True)
    inp = X.dyadic_inputs(gc)
    X.case_precondition(gc, inp)
    assert _plan(gc.case).S > 1
    A = _acts(inp["A"], torch.bfloat16, 0)
    gamma = torch.from_numpy(X.make_vec(1280, 5, 2.0 ** -4, 32)).to(torch.bfloat16).cuda()
    got = []
    for ms in (None, "1"):
        if ms:
            monkeypatch.setenv("B2_GEMM_TC_MAX_SPLIT", ms)
        op = _handle(gc, inp)
        res = Framed(M, 1280, torch.bfloat16, 4).fill(torch.from_numpy(inp["res"]).to(torch.bfloat16)).view
        ssq = torch.full((op.sumsq_parts(), M), -1.0, dtype=torch.float32, device="cuda")
        xg = torch.empty(M, 1280, dtype=torch.bfloat16, device="cuda")
        fr = Framed(M, 1280, torch.bfloat16, 4)
        ws = ops.Workspace()
        run = lambda: op(A, ws, out=fr.view, residual=res, sumsq_out=ssq, xg_out=(xg, gamma))
        run()
        torch.cuda.synchronize()
        one = (fr.view.clone(), xg.clone(), ssq.clone())
        ssq.fill_(-1.0)
        g = _graph(run)
        g.replay()
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(fr.view, one[0]) and torch.equal(xg, one[1]) and torch.equal(ssq, one[2])
        assert fr.guards_intact() and bool((ssq >= 0).all())
        got.append(one)
        monkeypatch.delenv("B2_GEMM_TC_MAX_SPLIT", raising=False)
    for a, b in zip(*got):
        assert torch.equal(a, b)
    y, E = X.restate(gc, inp)
    bad, _ = X.check(got[0][0].double().cpu().numpy(), y, E, "bf16")
    assert not bad.any()
    tiles = (got[0][0].double().cpu().numpy() ** 2).reshape(M, -1, 128).sum(-1).T
    assert np.allclose(got[0][2].double().cpu().numpy(), tiles, rtol=2.0 ** -20, atol=0)


@pytest.mark.parametrize("M", [17, 32, 64, 80])
@pytest.mark.parametrize("shape", [(3584, 18944, True), (3584, 18944, False)], ids=["pair", "multi"])
def test_halves_bit_identical_on_random_inputs(M, shape, monkeypatch):
    """Random bf16 activations (no exactness): the split leftovers carry the one accumulator chain of a whole n-group, so
    the output equals B2_GEMM_TC_MAX_SPLIT=1's bit for bit, over repeated launches and graph replays."""
    from b200spark import ops
    K, N, pair = shape
    gc = X.GpuCase("bal-random", X.Case(4, K, N, pair=pair), M, "tc", J=2)
    inp = X.dyadic_inputs(gc)
    assert _plan(gc.case).h > 0
    g = torch.Generator(device="cuda").manual_seed(M)
    A = (torch.randn(M, K, device="cuda", generator=g) * 0.5).to(torch.bfloat16)
    outs = []
    for ms in (None, "1"):
        if ms:
            monkeypatch.setenv("B2_GEMM_TC_MAX_SPLIT", ms)
        op = _handle(gc, inp)
        ws = ops.Workspace()
        run = lambda out: op(A, ws, out=out)
        first = run(torch.empty(M, N, dtype=torch.bfloat16, device="cuda"))
        out2 = torch.empty_like(first)
        gr = _graph(lambda: run(out2))
        for _ in range(3):
            run(first)
            gr.replay()
        torch.cuda.synchronize()
        assert torch.equal(out2, first)
        outs.append(first)
        monkeypatch.delenv("B2_GEMM_TC_MAX_SPLIT", raising=False)
    assert torch.equal(outs[0], outs[1])
    assert torch.isfinite(outs[0].float()).all()
