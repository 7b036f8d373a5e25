"""GPU: the GEMM's fused RMSNorm forms on exact-arithmetic inputs (tests/norm_exact.py), every output element held to the
restated arithmetic row by row instead of the 2e-2 of the random-row tests.

  * self-contained form (split-K GEMV, M <= 16): needle rows whose x^2 mass sits in one k-tile each (spread over every
    slice and staging chunk, the last row's in the K tail), gamma changing from tile to tile, staged products that round;
    cluster, global and forced splits; W4 / W8 / W16, per channel and g64 / g128, bf16 and fp16, SwiGLU pairs;
  * hand-off consumer (wgmma, M >= 17): statistics whose row m sits mostly in part m mod P; k-slices, whole rounds, carried
    n-groups, one slice, tail launches;
  * every row must match the restatement for ONE rs candidate (rsqrtf within 2 ulp, both evaluation forms): bit for bit for
    exact epilogues, inside check()'s bound widened over the candidates otherwise;
  * call forms: strided A and C, a guard frame, two runs and a graph replay bit-identical, the statistics untouched;
  * producer -> consumer chains: o_proj into gate+up, down into qkv and a W16 lm_head-shaped GEMM, the consumer restated
    from the xg and sumsq_out bits the producer wrote;
  * accuracy window: N(0,1) rows with one channel at 64 sigma, RMS 2^-16 .. 2^12, against an fp64 RMSNorm -> GEMM envelope,
    with the stand-alone b2_rmsnorm + GEMM measured beside it."""
import collections

import numpy as np
import pytest
import torch

import gemm_exact as X
import norm_exact as N
import test_gemm_exact_gpu as G

pytestmark = pytest.mark.gpu


def _gc(c):
    return X.GpuCase(c.id, c.case, c.M, c.path, env=c.env, bias=c.bias, res=c.res, act=c.act, alpha=c.alpha)


def _assert_path(gc, names, norm_self):
    want = X.launches(gc.case, gc.M, gc.env, G._sms(), norm_self=norm_self)
    assert {l["path"] for l in want} == {gc.path}, f"{gc.id}: the dispatch sends it to {want}"
    if names is None:
        return "dispatch copy"
    got = {n[n.index("wq_g"):n.index(">") + 1] for n in names}
    assert got <= {l["kernel"] for l in want}, f"{gc.id}: ran {sorted(got)}, expected {[l['kernel'] for l in want]}"
    return "profiler:" + ",".join(sorted(got))


def _match_rows(got, restate, cands, labels, ft, fused_forms):
    """Every row must agree with the restatement for one rs candidate (and one contraction form of the self epilogue).
    Returns (bad rows, per-row matching labels, worst deviation in bounds)."""
    M = got.shape[0]
    ys = [(lab, f, *restate(cands[:, i], f)) for i, lab in enumerate(labels) for f in fused_forms]
    exact = all(not E.any() for _, _, _, E in ys)
    if exact:
        ok = np.zeros((M, len(ys)), bool)
        for j, (_, _, y, _) in enumerate(ys):
            ok[:, j] = (X.rn_ft(y, ft) == got).all(1)
        matches = [[(ys[j][0], ys[j][1]) for j in range(len(ys)) if ok[m, j]] for m in range(M)]
        devs = np.stack([(np.abs(got - y) / X.bound_units(y, 0 * y, ft)).max(1) for _, _, y, _ in ys], 1)
        matched = np.where(ok, devs, np.inf).min(1)[ok.any(1)]              # each row at the candidate it matched
        dev = float(matched.max()) if matched.size else float("inf")
        return [m for m in range(M) if not ok[m].any()], matches, dev
    lo = np.min([y - E for _, _, y, E in ys], 0)
    hi = np.max([y + E for _, _, y, E in ys], 0)
    y, E = (lo + hi) / 2, (hi - lo) / 2
    bad, dev = X.check(got, y, E, ft)
    return sorted(set(np.argwhere(bad)[:, 0].tolist())), None, float(dev.max())


def _offsets(matches):
    """Distribution of the rs candidate each row matched (the one closest to the correctly rounded value if several do)."""
    h = collections.Counter()
    for ms in matches or []:
        if len(ms) == 0:
            continue
        rs_labels = {m[0] for m in ms}
        h["ambiguous" if len(rs_labels) == len(N.rs_candidates(np.zeros(1), 1)[1]) else
          "%s%+d" % min(rs_labels, key=lambda l: (abs(l[1]), l[0] != "sep"))] += 1
    return dict(h)


def _graph_equal(run, fr_args, first):
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    fr2 = G.Framed(*fr_args)
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            run(fr2.view)
    torch.cuda.current_stream().wait_stream(s)
    for _ in range(2):
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(fr2.view, first), "graph replay differs"
    assert fr2.guards_intact()


# ------------------------------------------------------------------------------------------------------------ self form
@pytest.mark.parametrize("i", range(len(N.SELF_CASES)), ids=lambda i: N.SELF_CASES[i].id)
def test_self_form(i, monkeypatch):
    sc = N.SELF_CASES[i]
    gc = _gc(sc)
    G._setenv(monkeypatch, gc)
    from b200spark import ops
    c = sc.case
    dt = G._dt(c)
    inp = N.self_inputs(sc)
    N.precondition_self(sc, inp)
    op = G._handle(gc, inp)
    pa, pc, off = X.call_form(i)
    x = G._acts(inp["x"], dt, pa)
    gamma = torch.from_numpy(inp["gamma"]).to(dt).cuda()
    ws = ops.Workspace()
    fr = G.Framed(sc.M, c.N, dt, pc, off)
    res = G.Framed(sc.M, c.N, dt, pc, off).fill(torch.from_numpy(inp["res"]).to(dt)).view if sc.res else None
    run = lambda out: op(x, ws, out=out, act=sc.act, alpha=sc.alpha, residual=res, norm_in=(None, gamma, c.K, N.EPS))
    how = _assert_path(gc, G._kernels(lambda: run(fr.view)), norm_self=True)
    split = G._gemv_split(gc, op, inp, monkeypatch)
    if split.startswith("split=none"):   # no workspace: either one k-slice or clusters, which only '-cluster' cases prove
        monkeypatch.setenv("B2_GEMM_CLUSTER", "0")
        ws0 = G._handle(gc, inp).workspace_bytes(sc.M)
        monkeypatch.delenv("B2_GEMM_CLUSTER")
        assert ws0 == 16, f"{sc.id}: splits K with clusters off, so it runs the cluster split unnamed: call it '-cluster'"
        split = "split=none (S=1)"
    first = fr.view.clone()
    run(fr.view)
    torch.cuda.synchronize()
    assert torch.equal(fr.view, first), f"{sc.id}: second run differs"
    assert fr.guards_intact(), f"{sc.id}: a write outside [M, N]"
    _graph_equal(run, (sc.M, c.N, dt, pc, off), first)
    got = first.double().cpu().numpy()
    cands, labels = N.rs_candidates(N.self_sumsq(inp["x"]), c.K)
    fused = (False, True) if N.contractible(inp["bias"], inp["res"], sc.act) else (False,)
    bad, matches, dev = _match_rows(got, lambda rs, f: N.restate_self(sc, inp, rs=rs, fused=f), cands, labels, c.ft, fused)
    assert not bad, f"{sc.id}: rows {bad} match no rs candidate"
    forms = collections.Counter(f for ms in matches or [] for _, f in ms[:1])
    print(f"SELF {sc.id} via={how} {split} elements={got.size} worst={dev:.3f} rs={_offsets(matches)} "
          f"contracted={dict(forms)}")


# ------------------------------------------------------------------------------------------------------------ consumer
@pytest.mark.parametrize("i", range(len(N.CONSUMER_CASES)), ids=lambda i: N.CONSUMER_CASES[i].id)
def test_handoff_consumer(i, monkeypatch):
    cc = N.CONSUMER_CASES[i]
    gc = _gc(cc)
    G._setenv(monkeypatch, gc)
    from b200spark import ops
    c = cc.case
    dt = G._dt(c)
    inp = N.consumer_inputs(cc)
    N.precondition_consumer(cc, inp)
    plan = N.tc_plan(c, G._sms(), cc.env)
    op = G._handle(gc, inp)
    pa, pc, off = X.call_form(i)
    A = G._acts(inp["A"], dt, pa)
    stats = torch.from_numpy(inp["stats"]).cuda()
    stats0 = stats.clone()
    ws = ops.Workspace()
    fr = G.Framed(cc.M, c.N, dt, pc, off)
    res = G.Framed(cc.M, c.N, dt, pc, off).fill(torch.from_numpy(inp["res"]).to(dt)).view if cc.res else None
    run = lambda out: op(A, ws, out=out, act=cc.act, alpha=cc.alpha, residual=res, norm_in=(stats, None, cc.hidden, N.EPS))
    how = _assert_path(gc, G._kernels(lambda: run(fr.view)), norm_self=False)
    first = fr.view.clone()
    run(fr.view)
    torch.cuda.synchronize()
    assert torch.equal(fr.view, first), f"{cc.id}: second run differs"
    assert fr.guards_intact(), f"{cc.id}: a write outside [M, N]"
    _graph_equal(run, (cc.M, c.N, dt, pc, off), first)
    assert torch.equal(stats, stats0), f"{cc.id}: the consumer wrote its statistics"
    got = first.double().cpu().numpy()
    pre = [N.tc_diffs(c, inp["wt"], inp["A"], plan)] + ([N.tc_diffs(c, inp["wt2"], inp["A"], plan)] if c.pair else [])
    cands, labels = N.rs_candidates(N.consumer_ss(inp["stats"]), cc.hidden)
    bad, matches, dev = _match_rows(got, lambda rs, f: N.restate_consumer(cc, inp, plan, rs=rs, pre=pre), cands, labels,
                                    c.ft, (False,))
    assert not bad, f"{cc.id}: rows {bad} match no rs candidate"
    print(f"CONSUMER {cc.id} via={how} plan=(S={plan.S} rounds={plan.rounds} h={plan.h}) P={cc.P} elements={got.size} "
          f"worst={dev:.3f} rs={_offsets(matches)}")


# ------------------------------------------------------------------------------------------------------------ chains
@pytest.mark.parametrize("ch", N.CHAIN_CASES, ids=lambda c: c.id)
def test_handoff_chain(ch):
    """Producer (xg_out, sumsq_out, P = its n-groups, tail launches at M > 64) then consumer on exactly what it wrote: the
    producer's xg is rn(C * gamma_out) of its stored C and its statistics the per-tile sums of C^2; every consumer row
    equals the restatement from those bits for one rs candidate."""
    from b200spark import ops
    p, c = ch.prod, ch.cons
    dt = G._dt(p)
    inp = N.chain_inputs(ch)
    pin = inp["prod"]
    gp = X.GpuCase(ch.id + "-prod", p, ch.M, "tc", res=True)
    opp = G._handle(gp, pin)
    cc = N.chain_consumer(ch)
    gcc = _gc(cc)
    opc = G._handle(gcc, inp)
    assert opp.sumsq_parts() == p.NG
    A = torch.from_numpy(pin["A"]).to(dt).cuda()
    res = torch.from_numpy(pin["res"]).to(dt).cuda()
    gamma = torch.from_numpy(inp["gamma"]).to(dt).cuda()
    ssq = torch.full((opp.sumsq_parts(), ch.M), float("nan"), dtype=torch.float32, device="cuda")
    xg = torch.empty(ch.M, p.N, dtype=dt, device="cuda")
    ws = ops.Workspace()
    C = opp(A, ws, residual=res, sumsq_out=ssq, xg_out=(xg, gamma))
    fr = G.Framed(ch.M, c.N, dt, 4)
    run = lambda out: opc(xg, ws, out=out, norm_in=(ssq, None, p.N, N.EPS))
    how = _assert_path(gcc, G._kernels(lambda: run(fr.view)), norm_self=False)
    torch.cuda.synchronize()
    assert fr.guards_intact()
    Cg = C.double().cpu().numpy()
    xgh = xg.double().cpu().numpy()
    st = ssq.cpu().numpy()
    assert np.array_equal(xgh, X.rn_ft(Cg * inp["gamma"][None, :], p.ft)), f"{ch.id}: xg is not rn(C * gamma_out)"
    assert np.allclose(st.astype(np.float64), (Cg ** 2).reshape(ch.M, -1, X.KBN).sum(-1).T, rtol=2.0 ** -20, atol=0), \
        f"{ch.id}: sumsq_out is not the per-tile sum of C^2 in [parts][M]"
    cin = dict(A=xgh, stats=st, wt=inp["wt"], wt2=inp["wt2"], bias=inp["bias"], res=None)
    X.precondition(c, inp["wt"], xgh, "tc", W2wt=inp["wt2"])
    plan = N.tc_plan(c, G._sms())
    pre = [N.tc_diffs(c, inp["wt"], xgh, plan)] + ([N.tc_diffs(c, inp["wt2"], xgh, plan)] if c.pair else [])
    cands, labels = N.rs_candidates(N.consumer_ss(st), p.N)
    got = fr.view.double().cpu().numpy()
    bad, matches, dev = _match_rows(got, lambda rs, f: N.restate_consumer(cc, cin, plan, rs=rs, pre=pre), cands, labels,
                                    c.ft, (False,))
    assert not bad, f"{ch.id}: rows {bad} match no rs candidate"
    print(f"CHAIN {ch.id} via={how} P={p.NG} plan=(S={plan.S} rounds={plan.rounds} h={plan.h}) elements={got.size} "
          f"worst={dev:.3f} rs={_offsets(matches)}")


# ------------------------------------------------------------------------------------------------------------ accuracy window
SWEEP_K, SWEEP_N = 3584, 1024
SWEEP_EXPS = list(range(-16, 13, 2))


def _sweep_rows(M, ft, e, seed):
    """N(0,1) rows with channel 7 at 64 sigma, scaled by 2^e, as FT values."""
    r = np.random.default_rng(seed)
    x = r.standard_normal((M, SWEEP_K))
    x[:, 7] = 64.0
    dt = torch.float16 if ft == "fp16" else torch.bfloat16
    return torch.from_numpy(x * 2.0 ** e).to(dt).double().numpy()


def _envelope(x, gamma, W, ft):
    """fp64 RMSNorm -> GEMM and its envelope: half an FT ulp of the result, plus the staging rounding of x rs gamma
    (the FT unit roundoff, 2^-8 / 2^-11 relative, no absolute floor), plus fp32 accumulation (K u) and the rs / read-out
    roundings.  A worst-case linear sum: it bounds, but cannot single out, the loss of a few fp16 subnormal products."""
    rs = 1 / np.sqrt((x * x).mean(1) + N.EPS)
    a = x * rs[:, None] * gamma[None, :]
    y = a @ W
    mag = np.abs(a) @ np.abs(W)
    u_ft = 2.0 ** -8 if ft == "bf16" else 2.0 ** -11
    E = u_ft * mag + (SWEEP_K + 16) * 2.0 ** -24 * mag
    return y, 0.5 * X.ulp_ft(np.abs(y) + E, ft) + E


# The exponents of 2 of the row RMS the fused forms are checked over and stay inside the fp64 envelope (b2_gemm_fuse,
# include/b200spark.h).  -16 is the floor of the sweep, not a measured edge; fp16 above 2^8: max |x gamma| > 65504, the
# staged value is inf, those points are skipped.
WINDOW = {"bf16": (-16, 12), "fp16": (-16, 8)}


@pytest.mark.parametrize("ft", ["bf16", "fp16"])
@pytest.mark.parametrize("form", ["self", "handoff"])
def test_accuracy_window(form, ft):
    from b200spark import ops
    dt = torch.float16 if ft == "fp16" else torch.bfloat16
    M = 2 if form == "self" else 17
    case = X.Case(4, SWEEP_K, SWEEP_N, ft=ft)
    wt = X.make_weights(case, 11)
    W = X.path_weights(case, wt, "tc" if form == "handoff" else "gemv")
    gamma = torch.from_numpy(X.make_vec(SWEEP_K, 12, 2.0 ** -6, 96)).to(dt).double().numpy()
    gamma[gamma == 0] = 2.0 ** -6
    gc = X.GpuCase("sweep", case, M, "gemv" if form == "self" else "tc")
    op = G._handle(gc, dict(wt=wt, wt2=None, bias=None))
    ws = ops.Workspace()
    g_d = torch.from_numpy(gamma).to(dt).cuda()
    rows = []
    for e in SWEEP_EXPS:
        x = _sweep_rows(M, ft, e, 100 + e)
        if ft == "fp16" and np.abs(x * gamma[None, :]).max() > 65504:
            rows.append((e, None, None, None))
            continue
        xd = torch.from_numpy(x).to(dt).cuda()
        if form == "self":
            out = op(xd, ws, norm_in=(None, g_d, SWEEP_K, N.EPS))
        else:
            xg = torch.from_numpy(X.rn_ft(x * gamma[None, :], ft)).to(dt).cuda()
            stats = torch.from_numpy((x * x).reshape(M, -1, 128).sum(-1).T.astype(np.float32).copy()).cuda()
            out = op(xg, ws, norm_in=(stats, None, SWEEP_K, N.EPS))
        ref = op(ops.rmsnorm(xd, g_d, N.EPS), ws)
        torch.cuda.synchronize()
        y, env = _envelope(x, gamma, W, ft)
        fused = float((np.abs(out.double().cpu().numpy() - y) / env).max())
        alone = float((np.abs(ref.double().cpu().numpy() - y) / env).max())
        rows.append((e, fused, alone, np.sqrt((x * x).mean())))
    lo, hi = WINDOW[ft]
    for e, fused, alone, rms in rows:
        print(f"WINDOW {form} {ft} rms=2^{e:+d} fused/env={'overflow' if fused is None else f'{fused:.3f}'} "
              f"standalone/env={'-' if alone is None else f'{alone:.3f}'}")
    inside = [(e, f) for e, f, _, _ in rows if lo <= e <= hi and f is not None]
    assert len(inside) == len([e for e in SWEEP_EXPS if lo <= e <= hi]), f"{form} {ft}: overflow inside the window"
    assert all(f <= 1.0 for _, f in inside), f"{form} {ft}: outside the envelope inside the window: {inside}"
