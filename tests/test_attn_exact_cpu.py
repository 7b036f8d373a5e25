"""CPU: the exact-arithmetic restatement of SpanAttention (tests/attn_exact.py) is right, its precondition holds on every GPU
case, its bound is sharp (plausible kernel bugs miss it by >= 4 bounds), and the restated quantized tile math shows that
small V scales need the power of two KVTraits::kPExp folds into P' before the fp16 rounding."""
import math

import numpy as np
import pytest

import attn_exact as X
import attn_needles as A

SMS = 132  # H100 SXM; the precondition is split-free, the grid only decides which rows end in a cross-CTA merge


def _cases():
    return X.single_cases() + X.step_cases() + X.rounding_cases() + [
        X.Case("head64-14/2", X.NONE, X.BF16, 16, 14, 2, [1, 31, 32, 33, 1000], head=64, seed=400)]


def test_qk_scale_table():
    for j, v in X.QK_SCALES.items():
        assert X.exact_qk_scale(j) == v
        assert X.scale_log2(v) == 2.0 ** -j
    assert X.scale_log2(1.0 / math.sqrt(128)) != 2.0 ** round(math.log2(X.scale_log2(1.0 / math.sqrt(128))))


def test_case_coverage():
    cs = _cases()
    kinds = {(c.mode, c.dtype == X.FP16, c.form) for c in cs}
    assert kinds >= {(m, h, "single") for m in X.MODES for h in (False, True)}
    assert {(c.mode, c.form) for c in cs} >= {(m, f) for m in X.MODES for f in ("single", "chain", "tree")}
    assert {c.hpg for c in cs} >= {1, 4, 7, 8, 16} and {c.span for c in cs} == {16, 128}
    assert {c.q_len for c in cs if c.form == "chain"} == {2, 5, 16}
    merges = set()
    for lens, nH, nG, mp in A.merge_shape_cases(SMS):
        merges |= {bg.merge for bg in A.decompose(lens, nG, SMS, mp).bgs}
    assert merges == {"single", "direct", "two-level"}


@pytest.mark.parametrize("case", _cases(), ids=lambda c: c.name)
def test_restatement_and_precondition(case):
    """The exact value agrees with fp64 softmax(qk_scale q K^T) V (natural units: qk_scale * log2 e is 2^-j up to the
    rounding of the fp32 product; rounding cases: up to the fp16 rounding of P'), the precondition holds (except on the
    rounding cases, which take the accumulation bound), and the bit prediction lies within the bound."""
    d = X.make(case)
    pre = X.precondition(case, d)
    assert pre < 1.0 or case.vbits, (case.name, pre)
    ex = X.exact(case, d)
    y = ex[0]
    alpha = case.qk_scale
    for b, tau, h, vis in X._row_sets(case):
        g = h // case.hpg
        K = d.kc[b][vis, g] * d.ks[b][vis, g, None]
        V = d.vc[b][vis, g] * d.vs[b][vis, g, None]
        s = alpha * (K @ d.q[b * case.q_len + tau, h])
        p = np.exp(s - s.max())
        ref = p @ V / p.sum()
        tol = 1e-5 * np.abs(V).max() + (2.0 ** -11 * (p @ np.abs(V)) / p.sum() if case.vbits else 0.0)
        assert (np.abs(ref - y[b * case.q_len + tau, h]) <= tol).all(), (case.name, b, tau, h)
    pred = X.predict(case, d, SMS, ex)
    assert (np.abs(pred - y) <= X.bound(case, y)).all()


@pytest.mark.parametrize("case", [c for c in _cases() if c.head == X.HEAD] + X.merge_cases(SMS), ids=lambda c: c.name)
def test_tile_restatement_predicts_the_bits(case):
    """The restatement per piece, tile and warp slice (running max, corr, l, o, cacc, warp merge, partial slots, cross-CTA
    merge) gives the predicted bits wherever no sum rounds, and lies within the bound on the rounding cases"""
    d = X.make(case)
    ex = X.exact(case, d)
    pred, ts = X.predict(case, d, SMS, ex), X.tile_sim(case, d, SMS)
    if case.vbits:
        assert (np.abs(ts - ex[0]) <= X.case_bound(case, d, SMS, ex[0])).all()
    else:
        assert np.array_equal(ts, pred), int((ts != pred).sum())


# ------------------------------------------------------------------------------------------------------- mutants
def _mutant(case, d, what):
    """the output of a kernel with one plausible bug, restated on the case's exact data"""
    m = X.Data(d.q.copy(), [x.copy() for x in d.kc], [x.copy() for x in d.ks], d.ku, d.kz,
               [x.copy() for x in d.vc], [x.copy() for x in d.vs], d.vu, d.vz)
    if what == "V params of tokens 2t and 2t+1 swapped":
        for b in range(len(case.lens)):
            n = m.vs[b].shape[0] // 2 * 2
            zc = d.vu[b] - d.vc[b] if case.mode in (X.I8, X.U4) else None
            m.vs[b][:n] = m.vs[b][:n].reshape(-1, 2, case.nG)[:, ::-1].reshape(n, case.nG)
            if zc is not None:  # the zero moves with the scale: c = u - z' with z' of the neighbour
                z = d.vz[b].copy()
                z[:n] = z[:n].reshape(-1, 2, case.nG)[:, ::-1].reshape(n, case.nG)
                m.vc[b] = d.vu[b] - z[..., None]
    elif what == "K scale read one token off at a param-chunk edge":
        for b in range(len(case.lens)):
            L = m.ks[b].shape[0]
            odd = np.arange(1, L - 1, 2)
            m.ks[b][odd] = d.ks[b][odd + 1]
    elif what == "Q and K d-orders disagree on one pair":
        m.q[..., [0, 1, 32, 33]] = d.q[..., [32, 33, 0, 1]]
    elif what == "V scale off by one token":
        for b in range(len(case.lens)):
            m.vs[b][:-1] = d.vs[b][1:]
    y = X.exact(case, m)[0]
    return X.rn_ft(y, case.dtype)


MUTANTS = ["V params of tokens 2t and 2t+1 swapped", "K scale read one token off at a param-chunk edge",
           "Q and K d-orders disagree on one pair", "V scale off by one token"]


@pytest.mark.parametrize("what", MUTANTS)
def test_mutants_miss_the_bound(what):
    """Each mutant misses the bound by >= 4 bounds on every GPU case of its mode (head-128 quantized caches for the
    parameter mutants, every case for the d-order)"""
    least = math.inf
    for case in _cases():
        if what != "Q and K d-orders disagree on one pair" and case.mode == X.NONE:
            continue
        if case.head != X.HEAD:
            continue
        d = X.make(case)
        y = X.exact(case, d)[0]
        r = float((np.abs(_mutant(case, d, what) - y) / X.bound(case, y)).max())
        least = min(least, r)
        assert r >= 4.0, (what, case.name, r)
    print("%-48s misses the bound by %.0f bounds (least over the cases)" % (what, least))


def test_head64_skipping_a_token_misses_the_bound():
    """head 64 dropping the last token of a partial 32-token step (lengths 31, 33, 1000)"""
    case = X.Case("head64-14/2", X.NONE, X.BF16, 16, 14, 2, [1, 31, 32, 33, 1000], head=64, seed=400)
    d = X.make(case)
    y = X.exact(case, d)[0]
    short = X.Case(**{**case.__dict__, "name": "head64-short"})
    short.visible = lambda b, tau: np.arange(case.lens[b]) < case.lens[b] - (1 if case.lens[b] % 32 and case.lens[b] > 1 else 0)
    ys = X.exact(short, d)[0]
    r = min(float((np.abs(X.rn_ft(ys, case.dtype) - y) / X.bound(case, y))[b].max()) for b in (1, 3, 4))
    print("head 64 skipping the last token of a partial step misses the bound by %.0f bounds" % r)
    assert r >= 4.0


def test_fp16_output_through_bf16_misses_the_bound():
    worst = math.inf
    for case in _cases():
        if case.dtype != X.FP16:
            continue
        d = X.make(case)
        y = X.exact(case, d)[0]
        r = float((np.abs(X.rn_ft(X.rn_ft(y, X.BF16), X.FP16) - y) / X.bound(case, y)).max())
        worst = min(worst, r)
        assert r >= 4.0, (case.name, r)
    print("fp16 output rounded through bf16 misses the bound by %.0f bounds" % worst)


TILE_MUTANTS = {
    # mutant: (cases it is applied to, cases on which it must miss by >= 4 bounds)
    "cacc not rescaled by corr": (lambda c: c.mode in (X.I8, X.U4), lambda c: c.form == "single" and c.dtype == X.BF16 and not c.vbits
                                  and not c.name.startswith("merge")),
    "zero-point term from unrounded P'": (lambda c: c.mode in (X.I8, X.U4), lambda c: c.vbits > 0),
    "merge weights from the other slot parity": (lambda c: c.name.startswith("merge"), lambda c: c.name.startswith("merge1")),
}


@pytest.mark.parametrize("what", list(TILE_MUTANTS))
def test_tile_mutants_miss_the_bound(what):
    """Bugs of the tile math and the merges, applied to the tile-level restatement on the GPU cases' inputs, against the
    bound each case is held to.  Where the inputs cannot show a mutant it is reported, not asserted: the zero-point term
    from unrounded P' needs P' to round (power-of-two V scales keep it exact), cacc without corr needs the running max to
    rise inside a warp's slices after a zero-point sum, and the slot parity needs a CTA whose other slot holds a partial."""
    applies, must = TILE_MUTANTS[what]
    seen = {}
    for case in [c for c in _cases() if c.head == X.HEAD] + X.merge_cases(SMS):
        if not applies(case):
            continue
        d = X.make(case)
        y = X.exact(case, d)[0]
        r = float((np.abs(X.tile_sim(case, d, SMS, what) - y) / X.case_bound(case, d, SMS, y)).max())
        seen[case.name] = r
        if must(case):
            assert r >= 4.0, (what, case.name, r)
    print("%-42s misses the bound by: %s" % (what, ", ".join("%s %.3g" % kv for kv in seen.items())))
    assert any(must(c) for c in [c for c in _cases() if c.head == X.HEAD] + X.merge_cases(SMS) if applies(c))


# ---------------------------------------------------------------------------------------------- V-scale sweep
def _sweep(mode, vexp, p_exp, seed):
    rng = np.random.default_rng(seed)
    L, hpg = 2048, 7
    k = A.to_type(rng.standard_normal((L, 128)), X.BF16)
    v = rng.standard_normal((L, 128))
    v = A.to_type(v * (2.0 ** vexp / np.abs(v).max(-1, keepdims=True)), X.BF16)
    q = A.to_type(rng.standard_normal((hpg, 128)), X.BF16)
    kc, ks = A.quantize(k, mode)
    vc, vs = A.quantize(v, mode)
    alpha = 1.0 / math.sqrt(128)
    vis = np.ones((hpg, L), bool)
    ref, env = X.envelope(mode, X.BF16, q, kc, ks, vc, vs, np.zeros(L), vis, alpha, 16)
    got = X.tile_math(mode, q, kc, ks, vc, vs, vis, alpha, p_exp)
    return float((np.abs(got - ref) / env).max())


@pytest.mark.parametrize("mode", [X.I8, X.U4, X.FP8], ids=lambda m: X.NAMES[m])
def test_v_scale_sweep_restated(mode):
    """P' = rn_f16(P s_v): fails the envelope at small V in int8 and fp8 (fp16 subnormals).  P' = rn_f16(P s_v 2^kPExp): passes over the
    window of include/b200spark.h, per-row max|v| in [2^-8, 2^12]."""
    before, after = {}, {}
    for vexp in range(-12, 13, 2):
        before[vexp] = _sweep(mode, vexp, 0, 20 + vexp)
        after[vexp] = _sweep(mode, vexp, X.P_EXP[mode], 20 + vexp)
    print("%s worst error/envelope by log2 max|v|:" % X.NAMES[mode])
    print("  k      " + " ".join("%6d" % k for k in before))
    print("  before " + " ".join("%6.2f" % before[k] for k in before))
    print("  after  " + " ".join("%6.2f" % after[k] for k in after))
    if mode != X.U4:  # u4's scale is ~17x int8's for the same rows: its P' stays normal over the sweep
        assert max(before[k] for k in before if k <= -6) > 1.0, before
    assert all(after[k] <= 1.0 for k in after if -8 <= k <= 12), after
