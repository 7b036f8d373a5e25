"""CPU checks of tests/norm_exact.py, the restatement behind test_norm_exact_gpu.py: it agrees with fp64 RMSNorm -> GEMM, its
exactness precondition holds for every GPU case, every GPU case reaches the kernel it names, and each of a list of
plausible kernel bugs, applied to the restatement, misses the GPU assertions by at least TEETH bounds on some GPU case."""
import numpy as np
import pytest

import gemm_exact as X
import norm_exact as N

TEETH = 4.0
SELF = {c.id: c for c in N.SELF_CASES}
CONS = {c.id: c for c in N.CONSUMER_CASES}
_inputs = {}


def _inp(c):
    if c.id not in _inputs:
        _inputs[c.id] = N.self_inputs(c) if isinstance(c, N.SelfCase) else N.consumer_inputs(c)
    return _inputs[c.id]


def _teeth(y, E, y_mut, ft):
    d = np.abs(y_mut - y) / X.bound_units(y, E, ft)
    return float(np.where(np.isnan(d), np.inf, d).max())


@pytest.mark.parametrize("cid", ["self-w4-pc-m3-k1000", "self-w4-g64-m9-k1088-fp16", "self-w16-m3-k1000", "self-pair-m9"])
def test_self_restatement_matches_fp64(cid):
    """The self form is fp64 RMSNorm (rs from sum x^2, no fp32 rounding) -> GEMM on the staged a' up to the roundings of rs
    and of the fp32 epilogue: a relative 2^-21 of sum |a' W| rs."""
    sc = SELF[cid]
    inp = _inp(sc)
    c = sc.case
    a = N.staged(inp["x"], inp["gamma"], c.ft)
    rs64 = 1 / np.sqrt((inp["x"] ** 2).mean(1) + N.EPS)
    W = X.dequant_exact(c, inp["wt"])
    y, E = N.restate_self(sc, inp)
    if c.pair:
        ref, _ = X.swiglu(sc.alpha * rs64[:, None] * (a @ W), sc.alpha * rs64[:, None] * (a @ X.dequant_exact(c, inp["wt2"])))
        tol = 2.0 ** -20 * np.abs(ref) + E
    else:
        ref, _ = X.expected(a * rs64[:, None], W, sc.act, sc.alpha, inp["bias"], inp["res"])
        mag = (np.abs(a) @ np.abs(W)) * rs64[:, None] * abs(sc.alpha)
        tol = 2.0 ** -21 * (mag + np.abs(ref)) + E + (2.0 ** -23 * np.abs(inp["res"]) if inp["res"] is not None else 0)
    assert np.all(np.abs(y - ref) <= tol)


@pytest.mark.parametrize("cid", ["cons-w4-pc-m33-fp16", "cons-w8-m20", "cons-w16-lmhead-m17", "cons-tail100", "cons-tail65"])
def test_consumer_restatement_matches_fp64(cid):
    """The consumer is fp64 (A (x) W) * rsqrt(sum stats / hidden + eps) up to the fp32 read-out, slice sum and epilogue
    roundings (grouped weights: the wgmma path's FT-rounded weights)."""
    cc = CONS[cid]
    inp = _inp(cc)
    c = cc.case
    plan = N.tc_plan(c)
    rs64 = 1 / np.sqrt(inp["stats"].astype(np.float64).sum(0) / cc.hidden + N.EPS)
    W = X.path_weights(c, inp["wt"], "tc")
    y, E = N.restate_consumer(cc, inp, plan)
    if c.pair:
        ref, _ = X.swiglu(cc.alpha * rs64[:, None] * (inp["A"] @ W), cc.alpha * rs64[:, None] * (inp["A"] @ X.path_weights(c, inp["wt2"], "tc")))
        tol = 2.0 ** -19 * np.abs(ref) + E
    else:
        ref, _ = X.expected(inp["A"] * rs64[:, None], W, cc.act, cc.alpha, inp["bias"], inp["res"])
        mag = (np.abs(inp["A"]) @ np.abs(W)) * rs64[:, None]
        tol = (plan.S + 3) * 2.0 ** -23 * (mag + np.abs(ref)) + E + (2.0 ** -23 * np.abs(inp["res"]) if inp["res"] is not None else 0)
    assert np.all(np.abs(y - ref) <= tol)


def test_rs_candidates_bracket_the_true_value():
    """The candidate set holds the correctly rounded 1/sqrt(t) of both forms and 2 ulp either side, zero rows included."""
    ss = np.array([0.0, 1e-9 * 3584, 3584.0, 12345.678, 2.0 ** 40], np.float32).astype(np.float64)
    cands, labels = N.rs_candidates(ss, 3584)
    assert cands.shape == (5, 10) and labels[2] == ("sep", 0)
    for m in range(5):
        true = 1 / np.sqrt(ss[m] / 3584 + 1e-6)
        assert cands[m].min() < true < cands[m].max()
        assert abs(cands[m, 2] - true) <= 2.0 ** -24 * true * 1.0001


@pytest.mark.parametrize("sc", N.SELF_CASES, ids=lambda c: c.id)
def test_self_precondition_holds(sc):
    N.precondition_self(sc, _inp(sc))


@pytest.mark.parametrize("cc", N.CONSUMER_CASES, ids=lambda c: c.id)
def test_consumer_precondition_holds(cc):
    N.precondition_consumer(cc, _inp(cc))


@pytest.mark.parametrize("ch", N.CHAIN_CASES, ids=lambda c: c.id)
def test_chain_precondition_holds(ch):
    """The producer's C = rn(res + W[k_m]) is exact (at most 5 significant bits), so xg = C * gamma_out is too, and the
    consumer's exactness precondition holds on it; the consumer sees P = the producer's n-groups and hidden = its N."""
    inp = N.chain_inputs(ch)
    pin = inp["prod"]
    y = pin["A"] @ X.dequant_exact(ch.prod, pin["wt"]) + pin["res"]
    assert np.array_equal(X.rn_ft(y, ch.prod.ft), y)
    xg = y * inp["gamma"][None, :]
    assert np.array_equal(X.rn_ft(xg, ch.prod.ft), xg)
    X.precondition(ch.cons, inp["wt"], xg, "tc", W2wt=inp["wt2"])
    cc = N.chain_consumer(ch)
    assert cc.P == ch.prod.NG and cc.hidden == ch.prod.N == ch.cons.K
    for c in (ch.prod, ch.cons):
        assert {l["path"] for l in X.launches(c, ch.M)} == {"tc"}


def test_every_case_reaches_its_kernel():
    for sc in N.SELF_CASES:
        ls = X.launches(sc.case, sc.M, sc.env, norm_self=True)
        assert {l["path"] for l in ls} == {"gemv"} and sc.M <= X.GEMV_MAX_M, sc.id
    # dense bf16 at M <= 16 goes to gemv2 unless the self form asks for the split-K kernel
    cb = {"B2_GEMV2_CB": "16"}
    assert X.launches(X.Case(16, 1000, 1024), 3, cb)[0]["path"] == "gemv2"
    assert X.launches(X.Case(16, 1000, 1024), 3, cb, norm_self=True)[0]["path"] == "gemv"
    plans = set()
    for cc in N.CONSUMER_CASES:
        ls = X.launches(cc.case, cc.M, cc.env)
        assert {l["path"] for l in ls} == {"tc"} and cc.M >= X.TC_MIN_M, cc.id
        assert len(ls) == (cc.M + 63) // 64
        p = N.tc_plan(cc.case, env=cc.env)
        plans.add("slices" if p.S > 1 else "carry" if p.h else "rounds" if p.rounds else "one")
    assert plans == {"slices", "carry", "one"}, plans


def test_rows_differ_where_the_kernels_pair_them():
    """Adjacent rows, rows m / m + 8 and m / m + 64 have different statistics; a zero row, a row far below eps and one
    about eps exist in every case with 8 rows or more."""
    for sc in N.SELF_CASES:
        ss = N.self_sumsq(_inp(sc)["x"])
        for d in (1, 8):
            nz = (ss[:-d] > 0) & (ss[d:] > 0)
            assert np.all(ss[:-d][nz] != ss[d:][nz]), sc.id
        if sc.M >= 8:
            ms = ss / sc.case.K
            assert ms[5] == 0 and ms[6] < 1e-3 * N.EPS and N.EPS / 30 < ms[7] < 30 * N.EPS, (sc.id, ms[5:8])
    for cc in N.CONSUMER_CASES:
        ss = N.consumer_ss(_inp(cc)["stats"])
        for d in (1, 8, 64):
            if cc.M > d:
                nz = (ss[:-d] > 0) & (ss[d:] > 0)
                assert np.all(ss[:-d][nz] != ss[d:][nz]), (cc.id, d)
        st = _inp(cc)["stats"]
        m = np.arange(cc.M)[ss > 0]
        assert np.all(st[m % cc.P, m] >= 0.5 * ss[m]), cc.id        # needle: part m mod P holds most of row m


# ------------------------------------------------------------------------------------------------------------ sharpness
def _self_margin(ids, mut):
    best = 0.0
    for cid in ids:
        sc = SELF[cid]
        inp = _inp(sc)
        y, E = N.restate_self(sc, inp)
        ym, _ = N.restate_self(sc, inp, mut=mut)
        best = max(best, _teeth(y, E, ym, sc.case.ft))
    return best


def _cons_margin(ids, mut):
    best = 0.0
    for cid in ids:
        cc = CONS[cid]
        inp = _inp(cc)
        plan = N.tc_plan(cc.case, env=cc.env)
        pre = [N.tc_diffs(cc.case, inp["wt"], inp["A"], plan)] + ([N.tc_diffs(cc.case, inp["wt2"], inp["A"], plan)] if cc.case.pair else [])
        y, E = N.restate_consumer(cc, inp, plan, pre=pre)
        ym, _ = N.restate_consumer(cc, inp, plan, pre=pre, mut=mut)
        best = max(best, _teeth(y, E, ym, cc.case.ft))
    return best


SMALL_SELF = ["self-w4-pc-m3-k1000", "self-w4-g64-m9-k1088-fp16", "self-w8-pc-m16-k1088", "self-w16-m16-fp16",
              "self-w4-pc-m9-forced3-fp16", "self-w4-pc-m16-silu", "self-pair-m9"]
SMALL_CONS = ["cons-w4-pc-m33-fp16", "cons-w8-m20", "cons-tail65", "cons-tail100", "cons-tail128-fp16", "cons-g128-pair",
              "cons-w16-m64-fp16"]

MUTATIONS = [
    # (number, description, form, mutation, cases)
    (1, "row m+1's rs (read-out pair swapped)", "cons", ("swap", None), SMALL_CONS),
    (2, "tail launch reads the rows 64 above", "cons", ("drop_m0", None), ["cons-tail65", "cons-tail100", "cons-tail128-fp16"]),
    (2, "norm_ld = 64 instead of M", "cons", ("ld64", None), ["cons-tail65", "cons-tail100", "cons-tail128-fp16"]),
    (3, "part 0 counted twice", "cons", ("part0_twice", None), SMALL_CONS),
    (4, "eps dropped (consumer)", "cons", ("eps_drop", None), SMALL_CONS),
    (4, "eps added after the rsqrt (consumer)", "cons", ("eps_after", None), SMALL_CONS),
    (4, "eps dropped (self)", "self", ("eps_drop", None), SMALL_SELF),
    (4, "eps added after the rsqrt (self)", "self", ("eps_after", None), SMALL_SELF),
    (6, "sum (x gamma)^2 instead of sum x^2", "self", ("ss_xg", None), SMALL_SELF),
    (7, "zero-point row sums from x", "self", ("suma_x", None), SMALL_SELF),
    (7, "zero-point row sums from unrounded x gamma", "self", ("suma_unrounded", None), SMALL_SELF),
    (9, "staging kept unrounded", "self", ("unrounded", None), SMALL_SELF),
    (10, "SwiGLU: rs on the gate only (self)", "self", ("gate_only", None), ["self-pair-m9"]),
    (10, "SwiGLU: rs on the gate only (consumer)", "cons", ("gate_only", None), ["cons-g128-pair"]),
    (11, "carried n-group scaled twice", "cons", ("carry_twice", None), ["cons-w4-pc-m64-multi"]),
]


@pytest.mark.parametrize("mi", range(len(MUTATIONS)), ids=lambda i: f"m{MUTATIONS[i][0]}-{MUTATIONS[i][3][0]}")
def test_mutation_misses_by_teeth(mi):
    no, desc, form, mut, ids = MUTATIONS[mi]
    margin = (_self_margin if form == "self" else _cons_margin)(ids, mut)
    print(f"MUTATION {no} {desc}: {margin:.1f} bounds")
    assert margin >= TEETH, (desc, margin)


@pytest.mark.parametrize("P", [1, 3, 8, 28, 64])
def test_mutation_every_dropped_part_is_seen(P):
    """Mutation 3: whichever statistics part is dropped, some case with P parts misses by TEETH."""
    ids = [c.id for c in N.CONSUMER_CASES if c.P == P and c.case.K <= 2048 or c.P == P and c.id == "cons-w4-pc-m32-o"]
    assert ids, P
    worst = min(_cons_margin(ids, ("drop_part", p)) for p in range(P))
    print(f"MUTATION 3 one of {P} parts dropped: >= {worst:.1f} bounds")
    assert worst >= TEETH


@pytest.mark.parametrize("S", [2, 3, 4, 5, 8])
def test_mutation_every_dropped_slice_is_seen(S):
    """Mutation 5: whichever k-slice's sum x^2 is left out of the reduction, some case misses by TEETH."""
    worst = np.inf
    for s in range(S):
        best = 0.0
        for cid in SMALL_SELF:
            sc = SELF[cid]
            sl = N.gemv_slices(sc.case, S)[s]
            best = max(best, _self_margin([cid], ("drop_slice", sl)))
        worst = min(worst, best)
    print(f"MUTATION 5 one of {S} slices dropped: >= {worst:.1f} bounds")
    assert worst >= TEETH


@pytest.mark.parametrize("chunk_tiles", [2, 4, 8, 16])
def test_mutation_gamma_from_previous_chunk(chunk_tiles):
    """Mutation 8: gamma read from the staging chunk before (chunk lengths the plan can choose)."""
    margin = _self_margin(SMALL_SELF, ("gamma_prev", chunk_tiles * X.KBK))
    print(f"MUTATION 8 gamma from the previous {chunk_tiles}-tile chunk: {margin:.1f} bounds")
    assert margin >= TEETH
