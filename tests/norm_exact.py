"""Exact-arithmetic inputs and a restatement of the weight-only GEMM's two fused RMSNorm forms (b2_gemm_fuse), so a test can
hold every output element to the rounding of the restated arithmetic instead of the 2e-2 of the random-row tests.
Builds on tests/gemm_exact.py (cases, weights, precondition, check) and tests/tc_schedule.py (the wgmma plan).

Importable without the native library or a GPU.

Self-contained form (split-K GEMV, M <= 16; wq_gemm.cu, norm_self): the kernel stages a' = rn_FT(x * gamma) (the product of
two FT values is exact in fp32: one rounding), takes the zero-point row sums from a', collects ss = sum x^2 from the
unscaled x, reduces the exact fp32 tile Q = a' (x) W over the k-slices (cluster, global or forced split) and scales it:
  v = Q * fl(alpha * rs),  rs = rsqrtf(ss * fl(1 / K) + eps),  then + bias, activation, + residual, one FT store
  (SwiGLU: silu(Qg * fl(alpha rs)) * (Qu * fl(alpha rs))).
precondition_self() adds to the GEMM precondition (row by row: every row has its own grid) that sum x^2 is exact in fp32 in
every order the split forms add it (cluster ranks in order, the global split's lane butterfly, the per-chunk sums).

Hand-off consumer (wgmma, M >= 17; wq_gemm_tc.cu, norm_sumsq): ss = sum_p stats[p][m] summed in fp32 in p order (any fp32
statistics: numpy float32 repeats it bit for bit), rs as above with hidden for K, and at the accumulator read-out of every
k-slice
  part = fl(fl(sz * rs) * (d - z' sum a))      (dense and sub-channel weights: sz = 1, no zero-point term)
the partials summed in slice order for rounds == 0 plans (a whole or carried n-group is one partial: the head parks raw
accumulators), then alpha (a power of two here: exact), + bias, activation, + residual, one FT store.

rsqrtf is the one step a CPU cannot repeat: the CUDA Programming Guide gives it a maximum error of 2 ulp, and whether
ss * invH + eps is contracted into one FMA is the compiler's choice.  rs_candidates() returns, per row, the fp32 values
within 2 ulp of 1/sqrt(t) for t under both evaluation forms; a test asserts that ONE candidate per row makes every element of
the row agree with the restatement (exact epilogues: bit for bit), and records which candidate it was.  The self form's
v = Q * ra followed by + bias (or + residual) may also be contracted: both forms are restated (`fused`).
"""
from dataclasses import dataclass, field

import numpy as np

import gemm_exact as X
import tc_schedule as TS

EPS = 1e-6
ULPS = 2                     # rsqrtf maximum error (CUDA Programming Guide, mathematical functions appendix)
LD = np.longdouble


def f32(a):
    """Round to fp32, returned as fp64 (products of two fp32 values are exact in fp64, so f32(a * b) is one rounding)."""
    return np.asarray(a).astype(np.float32).astype(np.float64)


# --------------------------------------------------------------------------------------------------- 1 / rms
def t_forms(ss, hidden, eps=EPS):
    """The two fp32 values rsqrtf may be applied to: fl(fl(ss * invH) + eps) and the FMA form fl(ss * invH + eps)."""
    ss = f32(ss)
    invH = f32(1.0 / hidden)
    e = f32(eps)
    t_sep = f32(f32(ss * invH) + e)
    t_fma = np.asarray(LD(ss) * LD(invH) + LD(e)).astype(np.float32).astype(np.float64)
    return t_sep, t_fma


def rsqrt_rn(t):
    """Correctly rounded fp32 1 / sqrt(t)."""
    with np.errstate(divide="ignore"):
        return np.asarray(LD(1) / np.sqrt(np.asarray(t, LD))).astype(np.float32).astype(np.float64)


def rs_candidates(ss, hidden, eps=EPS, ulps=ULPS):
    """[M, C] candidate rs values and C labels (form, ulp offset from the correctly rounded 1 / sqrt(t) of that form)."""
    cands, labels = [], []
    for form, t in zip(("sep", "fma"), t_forms(ss, hidden, eps)):
        r = rsqrt_rn(t).astype(np.float32)
        for off in range(-ulps, ulps + 1):
            v = r.copy()
            for _ in range(abs(off)):
                v = np.nextafter(v, np.float32(np.inf if off > 0 else 0)).astype(np.float32)
            cands.append(v.astype(np.float64))
            labels.append((form, off))
    return np.stack(cands, 1), labels


def rs_nominal(ss, hidden, eps=EPS):
    return rsqrt_rn(t_forms(ss, hidden, eps)[0])


# --------------------------------------------------------------------------------------------------- epilogues
def finish(P, ra, bias=None, res=None, act=X.ACT_NONE, fused=False, Pu=None, ra_u=None):
    """fp32 epilogue of one tile P [M, N] (exact fp32 values) scaled by ra [M] (or a scalar): v = P * ra, + bias, act,
    + residual.  fused: v = fl(P * ra + first addend) (bias, else the residual of an activation-free epilogue).  Pu: the
    up half of a SwiGLU pair (scaled by ra_u, default ra).  Returns (y, E): y the value the kernel rounds to FT, E its fp32
    error bound (0: y is exact)."""
    ra = np.broadcast_to(np.asarray(ra, np.float64).reshape(-1, 1), (P.shape[0], 1))
    if Pu is not None:
        ru = ra if ra_u is None else np.broadcast_to(np.asarray(ra_u, np.float64).reshape(-1, 1), (P.shape[0], 1))
        return X.swiglu(f32(P * ra), f32(Pu * ru))
    first = bias[None, :] if bias is not None else (res if (res is not None and act == X.ACT_NONE) else None)
    if fused and first is not None:
        v = f32(np.asarray(LD(P) * LD(ra) + LD(first)))
        added_res = bias is None
    else:
        v = f32(P * ra)
        if bias is not None:
            v = f32(v + bias[None, :])
        added_res = False
    if act in X.EXACT_ACTS:
        y = f32(X._act(v, act))
        if res is not None and not added_res:
            y = f32(y + res)
        return y, np.zeros(y.shape)
    y = X._act(v, act)
    E = X.act_bound(v, y, act)
    return (y + res if res is not None else y), E


def contractible(bias, res, act):
    """Whether the self form's v = Q * ra has an addend the compiler may fuse into it."""
    return bias is not None or (res is not None and act == X.ACT_NONE)


# --------------------------------------------------------------------------------------------------- self-contained form
def staged(x, gamma, ft, rounded=True):
    """a' = rn_FT(x * gamma) (x, gamma: fp64 of FT values; their product is an fp32 number)."""
    p = x * np.asarray(gamma)[None, :]
    return X.rn_ft(p, ft) if rounded else p


def self_tile(case, wt, a, zsum=None):
    """Q = a (x) W exactly (fp64; an fp32 number under precondition_self).  zsum: the row sums the zero-point term is taken
    from, if not a (a mutation): Q - s z' (zsum - sum a) per quantization group."""
    Q = a @ X.dequant_exact(case, wt)
    if zsum is not None and case.wbits != 16:
        g = X.group_index(case)
        for gi in range(case.G):
            ks = g == gi
            zp = wt.z[gi] + _zbias(case)
            Q = Q - (zsum[:, ks].sum(1) - a[:, ks].sum(1))[:, None] * (zp * wt.s[gi])[None, :]
    return Q


def _zbias(case):
    return case.b0 if case.wbits == 4 else 17 * case.b0 + (128 if case.signed else 0)


def gemv_slices(case, S):
    """k ranges of the S k-slices of the split-K GEMV (quanta of group_tiles tiles split evenly)."""
    gt = case.group // X.KBK if case.grouped else 1
    quanta = case.KT // gt
    return [(s * quanta // S * gt * X.KBK, (s + 1) * quanta // S * gt * X.KBK) for s in range(S)]


def self_sumsq(x, mut=None):
    """sum x^2 per row (exact under the precondition).  mut: ('drop_slice', (k0, k1)) leaves a k range out."""
    sq = x * x
    if mut and mut[0] == "drop_slice":
        k0, k1 = mut[1]
        sq = sq.copy()
        sq[:, k0:k1] = 0
    return f32(sq.sum(1))


def restate_self(sc, inp, rs=None, fused=False, mut=None):
    """(y, E) of one self-form case; rs [M] (default: the correctly rounded separate form).  mut: a (name, arg) mutation."""
    c = sc.case
    x, gamma = inp["x"], inp["gamma"]
    name, arg = mut if mut else (None, None)
    g = gamma
    if name == "gamma_prev":                        # gamma of the chunk arg k before
        g = np.concatenate([gamma[:arg], gamma[:-arg]])
    a = staged(x, g, c.ft, rounded=name != "unrounded")
    if rs is None:
        ss = f32((a * a).sum(1)) if name == "ss_xg" else self_sumsq(x, mut if name == "drop_slice" else None)
        hid = c.K
        if name == "eps_drop":
            rs = rsqrt_rn(f32(ss * f32(1.0 / hid)))
        elif name == "eps_after":
            rs = f32(rsqrt_rn(f32(ss * f32(1.0 / hid))) + f32(EPS))
        else:
            rs = rs_nominal(ss, hid)
    if mut is None and "_tiles" in inp:          # the unmutated tiles do not depend on rs: computed once per case
        return _finish_self(sc, inp, inp["_tiles"], rs, fused, name)
    zsum = {"suma_x": x, "suma_unrounded": x * gamma[None, :]}.get(name)
    tiles = [self_tile(c, inp["wt"], a, zsum)] + ([self_tile(c, inp["wt2"], a, zsum)] if c.pair else [])
    if mut is None:
        inp["_tiles"] = tiles
    return _finish_self(sc, inp, tiles, rs, fused, name)


def _finish_self(sc, inp, tiles, rs, fused, name):
    ra = f32(sc.alpha * rs)
    if sc.case.pair:
        return finish(tiles[0], ra, Pu=tiles[1], ra_u=f32(sc.alpha + 0 * rs) if name == "gate_only" else None)
    return finish(tiles[0], ra, inp["bias"], inp["res"], sc.act, fused)


def precondition_self(sc, inp):
    """Raise ValueError unless the self form's arithmetic before the 1/rms scaling is exact for these inputs: x * gamma in
    fp32, sum x^2 in every order (every partial below 2^24 units of the row's grid), and the GEMM on a' row by row
    (gemm_exact.precondition).  Returns the worst partial sum in units of the limit."""
    c = sc.case
    x, gamma = inp["x"], inp["gamma"]
    if not X.is_f32(x * gamma[None, :]):
        raise ValueError("x * gamma is not an fp32 number")
    a = staged(x, gamma, c.ft)
    worst = 0.0
    for m in range(x.shape[0]):
        nz = np.abs(x[m][x[m] != 0])
        if nz.size:
            u = float(np.exp2(np.floor(np.log2(nz.min()))))
            while not np.all(np.mod(x[m] / u, 1.0) == 0):
                u /= 2
            sq = (x[m] / u) ** 2
            if sq.sum() >= 2.0 ** 24:
                raise ValueError(f"row {m}: sum x^2 reaches {sq.sum() / 2 ** 24:.2f} x 2^24 units")
            if np.any(a[m] != 0):
                worst = max(worst, X.precondition(c, inp["wt"], a[m:m + 1], "gemv", W2wt=inp["wt2"]))
    return worst


# --------------------------------------------------------------------------------------------------- hand-off consumer
def tc_plan(case, sms=X.H100_SMS, env=None):
    env = env or {}
    return TS.plan(case.NG, case.KT, sms, int(env.get("B2_GEMM_TC_MAX_SPLIT", TS.MAX_SPLIT)))


def tc_diffs(case, wt, A, plan):
    """The exact per-k-slice accumulator terms (d - z' sum a for per-channel weights, d for dense / sub-channel) and the
    scale that multiplies rs at the read-out (sz: the channel scale; 1 for dense / sub-channel)."""
    slices = X.tc_slices(case, plan.S) if plan.rounds == 0 else [(0, case.KT)]
    if case.wbits != 16 and not case.grouped:
        Wd, sz = (wt.q - wt.z[0][None, :]).astype(np.float64), wt.s[0]
    else:
        Wd, sz = X.path_weights(case, wt, "tc"), np.ones(case.N)
    out = []
    for kt0, kt1 in slices:
        k0, k1 = kt0 * X.KBK, min(kt1 * X.KBK, case.K)
        out.append(A[:, k0:k1] @ Wd[k0:k1])
    return out, sz


def tc_acc(diffs, sz, rs, carried=None):
    """The fp32 tile after the read-out and the slice-order sum, for rs [M].  carried: channel mask of n-groups scaled a
    second time (a mutation)."""
    sr = f32(sz[None, :] * rs[:, None])
    acc = None
    for d in diffs:
        part = f32(sr * d)
        if carried is not None:
            part = np.where(carried[None, :], f32(part * rs[:, None]), part)
        acc = part if acc is None else f32(acc + part)
    return acc


def consumer_ss(stats, mut=None):
    """sum_p stats[p][m] in fp32, p order; mut: ('drop_part', p), ('part0_twice', None), ('ld64', None)."""
    st = np.asarray(stats, np.float32)
    name, arg = mut if mut else (None, None)
    if name == "drop_part":
        st = np.delete(st, arg, axis=0)
    elif name == "part0_twice":
        st = np.concatenate([st[:1], st], axis=0)
    elif name == "ld64":          # norm_ld = 64 instead of M: row m of a launch at m0 reads flat[p * 64 + m0 + m]
        P, M = st.shape
        flat = np.concatenate([st.ravel(), np.zeros(P * 64, np.float32)])
        st = np.stack([flat[p * 64 + np.arange(M)] for p in range(P)])
    ss = np.zeros(st.shape[1], np.float32)
    for p in range(st.shape[0]):
        ss = (ss + st[p]).astype(np.float32)
    return ss.astype(np.float64)


def consumer_rs(cc, stats, mut=None):
    name, arg = mut if mut else (None, None)
    ss = consumer_ss(stats, mut if name in ("drop_part", "part0_twice", "ld64") else None)
    invH = f32(1.0 / cc.hidden)
    if name == "eps_drop":
        rs = rsqrt_rn(f32(ss * invH))
    elif name == "eps_after":
        rs = f32(rsqrt_rn(f32(ss * invH)) + f32(EPS))
    else:
        rs = rs_nominal(ss, cc.hidden)
    if name == "swap":                      # the read-out's ascale[m] / ascale[m + 1] pair swapped
        rs = rs[np.arange(len(rs)) ^ 1] if len(rs) % 2 == 0 else rs[np.minimum(np.arange(len(rs)) ^ 1, len(rs) - 1)]
    elif name == "drop_m0":                 # a tail launch reads the statistics of the rows 64 above
        rs = rs.copy()
        rs[64:] = rs[:len(rs) - 64]
    return rs


def carried_channels(case, plan):
    """Channel mask of the n-groups a split head / tail computes."""
    width = 64 if case.pair else X.KBN
    ng = np.arange(case.N) // width
    return (ng >= plan.nfull) if plan.h else np.zeros(case.N, bool)


def restate_consumer(cc, inp, plan, rs=None, pre=None, mut=None):
    """(y, E) of one consumer case for rs [M] (default: from the statistics, correctly rounded).  pre: tc_diffs of the
    weights (computed if not given)."""
    c = cc.case
    name = mut[0] if mut else None
    if rs is None:
        rs = consumer_rs(cc, inp["stats"], mut)
    if pre is None:
        pre = [tc_diffs(c, inp["wt"], inp["A"], plan)] + ([tc_diffs(c, inp["wt2"], inp["A"], plan)] if c.pair else [])
    carried = carried_channels(c, plan) if name == "carry_twice" else None
    acc = tc_acc(*pre[0], rs, carried)
    if c.pair:
        rs_u = np.ones_like(rs) if name == "gate_only" else rs
        return finish(acc, cc.alpha, Pu=tc_acc(*pre[1], rs_u, carried))
    return finish(acc, cc.alpha, inp["bias"], inp["res"], cc.act)


# --------------------------------------------------------------------------------------------------- GPU cases
@dataclass
class SelfCase:
    """One self-form GEMM (split-K GEMV): env knobs set before the handle is created; dens: nonzero fraction of a row
    outside its needle tile; J: largest |x| code."""
    id: str
    case: X.Case
    M: int
    env: dict = field(default_factory=dict)
    act: int = X.ACT_NONE
    alpha: float = 1.0
    bias: bool = False
    res: bool = False
    dens: float = 0.125
    J: int = 3
    path: str = "gemv"


@dataclass
class ConsumerCase:
    """One hand-off consumer GEMM (wgmma): P statistics parts of a hidden size `hidden`."""
    id: str
    case: X.Case
    M: int
    P: int
    env: dict = field(default_factory=dict)
    act: int = X.ACT_NONE
    alpha: float = 1.0
    bias: bool = False
    res: bool = False
    J: int = 3
    hidden: int = 3584
    path: str = "tc"


# row scales of the self form: adjacent rows differ by power-of-two and other factors, so do rows m, m + 8; row 5 is zero,
# row 6 has sum x^2 / K far below eps, row 7 about eps (self_inputs)
ROW_SCALE = [1.0, 3.0, 1.5, 0.625, 2.0, 0.0, 2.0 ** -14, 2.0 ** -7, 0.75, 3.5, 1.25, 0.5, 2.5, 1.75, 0.875, 3.0]
GAMMA_CYCLE = [1.0, 0.75, 1.5, 1.25, 0.625, 1.75, 0.875]   # 7 tiles: no chunk length repeats it


def _seed(id_):
    return sum(map(ord, id_))


def needle_tile(m, M, KT0):
    """The 64-k tile that carries most of row m's x^2: spread over K, the last row's in the K tail."""
    return KT0 - 1 if M == 1 else (m * (KT0 - 1)) // (M - 1)


def self_weights(case, seed):
    """gemm_exact.make_weights with scales 2^-ps or 2^-(ps+1): s (acc - z' sum a) stays exact for rows whose staged values
    carry up to 16 significant bits (the codes, zero points and dense weights are gemm_exact's)."""
    wt = X.make_weights(case, seed)
    if case.wbits != 16:
        ps = -int(np.log2(wt.unit_s)) - 2
        wt.s = np.exp2(-(ps + np.random.default_rng(seed + 7).integers(0, 2, size=wt.s.shape)))
        wt.unit_s = 2.0 ** -(ps + 1)
    return wt


def self_inputs(sc):
    """x [M, K] (FT values), gamma [K], weights, bias, residual of one self-form case.  Row m: sparse codes j in
    [-J, J] (density dens) plus a needle tile half filled with codes +-(2J+1), times ROW_SCALE[m] / 8.  gamma: one value of
    GAMMA_CYCLE per 64-k tile times (1, 1.25, 1.5, 1.75) by k mod 4, so x * gamma carries up to 14 significant bits."""
    c = sc.case
    r = np.random.default_rng(_seed(sc.id))
    K, M = c.K, sc.M
    KT0 = (K + X.KBK - 1) // X.KBK
    j = r.integers(-sc.J, sc.J + 1, size=(M, K)) * (r.random((M, K)) < sc.dens)
    for m in range(M):
        t = needle_tile(m, M, KT0)
        k0, k1 = t * X.KBK, min((t + 1) * X.KBK, K)
        j[m, k0:k1] = (2 * sc.J + 1) * r.choice([-1, 0, 0, 1], size=k1 - k0)
    scale = np.array([ROW_SCALE[m % len(ROW_SCALE)] for m in range(M)]) / 8
    if M > 7:                                       # row 7: sum x^2 / K about eps (a power of two near it)
        scale[7] = 2.0 ** np.round(np.log2(np.sqrt(EPS * K / (j[7] ** 2).sum())))
    x = j * scale[:, None]
    k = np.arange(K)
    gamma = np.array(GAMMA_CYCLE)[(k // X.KBK) % len(GAMMA_CYCLE)] * (1 + (k % 4) / 4)
    wt = self_weights(c, _seed(sc.id) + 1)
    wt2 = self_weights(c, _seed(sc.id) + 2) if c.pair else None
    bias = X.make_vec(c.N, _seed(sc.id) + 3) if sc.bias else None
    res = X.make_vec(M * c.N, _seed(sc.id) + 4).reshape(M, c.N) if sc.res else None
    return dict(x=x, gamma=gamma, wt=wt, wt2=wt2, bias=bias, res=res)


def consumer_inputs(cc):
    """A [M, K] (dyadic, gemm_exact.make_acts), statistics [P, M] fp32, weights, bias, residual.  Row m's sum of squares
    is concentrated in part m mod P (the other parts small, non-dyadic); the rows' mean squares step by non-power-of-two
    factors, row 5 is zero, row 6 far below eps, row 7 about eps."""
    c = cc.case
    r = np.random.default_rng(_seed(cc.id))
    M, P = cc.M, cc.P
    A = X.make_acts(M, c.K, cc.J, 3, _seed(cc.id) + 5)
    ms = 2.0 ** (((np.arange(M) * 7) % 23) / 4.0 - 3.0)         # mean squares 2^-3 .. 2^2.5 in 2^(1/4) steps
    ms[5 % M] = 0.0
    if M > 7:
        ms[6], ms[7] = 1e-9, 1e-6
    total = ms * cc.hidden
    w = r.uniform(0.002, 0.01, size=(P, M))
    w[np.arange(M) % P, np.arange(M)] = 1.0
    stats = (w / w.sum(0, keepdims=True) * total[None, :]).astype(np.float32)
    wt = X.make_weights(c, _seed(cc.id) + 1)
    wt2 = X.make_weights(c, _seed(cc.id) + 2) if c.pair else None
    bias = X.make_vec(c.N, _seed(cc.id) + 3) if cc.bias else None
    res = X.make_vec(M * c.N, _seed(cc.id) + 4).reshape(M, c.N) if cc.res else None
    return dict(A=A, stats=stats, wt=wt, wt2=wt2, bias=bias, res=res)


def precondition_consumer(cc, inp):
    return X.precondition(cc.case, inp["wt"], inp["A"], "tc", unit_a=2.0 ** -3, W2wt=inp["wt2"])


C = X.Case
QKV, O, GU = (3584, 4608), (3584, 3584), (3584, 18944)

SELF_CASES = [
    SelfCase("self-w4-pc-m1-qkv-cluster", C(4, *QKV), 1, bias=True),
    SelfCase("self-w4-pc-m2-gateup", C(4, *GU, pair=True), 2, dens=0.06),
    SelfCase("self-w4-pc-m3-k1000", C(4, 1000, 1024), 3, res=True, alpha=-0.75),
    SelfCase("self-w4-g128-m8-qkv-cluster", C(4, *QKV, group=128), 8, bias=True, res=True, dens=0.08),
    SelfCase("self-w4-g64-m9-k1088-fp16", C(4, 1088, 1000, group=64, ft="fp16"), 9, act=X.ACT_RELU, dens=0.02, J=1),
    SelfCase("self-w8-pc-m16-k1088", C(8, 1088, 1024), 16, alpha=0.5, bias=True, J=0),
    SelfCase("self-w16-m3-k1000", C(16, 1000, 1024), 3, res=True),
    SelfCase("self-w16-m16-fp16", C(16, 1088, 520, ft="fp16"), 16, bias=True, dens=0.02, J=1),
    SelfCase("self-w4-pc-m8-noclus", C(4, *QKV), 8, env={"B2_GEMM_CLUSTER": "0"}, res=True, dens=0.08),
    SelfCase("self-w4-g128-m16-noclus", C(4, *QKV, group=128), 16, env={"B2_GEMM_CLUSTER": "0"}, alpha=-1.0, dens=0.06),
    SelfCase("self-w4-pc-m2-forced5", C(4, 1000, 1024), 2, env={"B2_GEMM_FORCE_SPLIT": "5"}, bias=True),
    SelfCase("self-w4-pc-m9-forced3-fp16", C(4, 1088, 1024, ft="fp16"), 9, env={"B2_GEMM_FORCE_SPLIT": "3"}, res=True,
             dens=0.02, J=1),
    SelfCase("self-w4-pc-m16-silu", C(4, 1088, 1024), 16, act=X.ACT_SILU, bias=True, dens=0.08),
    SelfCase("self-w8-g128-m9-gelu", C(8, 1024, 640, group=128), 9, act=X.ACT_GELU_TANH, J=0),
    SelfCase("self-w4-pc-m1-qkv-fp16-cluster", C(4, *QKV, ft="fp16"), 1, bias=True, res=True, dens=0.02, J=1),
    SelfCase("self-pair-m9", C(4, 1088, 704, pair=True), 9, alpha=0.5),
    SelfCase("self-pair-m16-fp16", C(4, 1088, 704, pair=True, ft="fp16"), 16, dens=0.02, J=1),
]

CONSUMER_CASES = [
    ConsumerCase("cons-w4-pc-m17-qkv", C(4, *QKV), 17, 28, bias=True),
    ConsumerCase("cons-w4-pc-m32-o", C(4, *O), 32, 1, res=True),
    ConsumerCase("cons-w4-pc-m33-fp16", C(4, 1024, 1024, ft="fp16"), 33, 3, res=True, bias=True),
    ConsumerCase("cons-w4-pc-m64-gateup", C(4, *GU, pair=True), 64, 28, J=2),
    ConsumerCase("cons-w4-pc-m64-multi", C(4, *GU), 64, 8, act=X.ACT_SILU),
    ConsumerCase("cons-w4-g128-m64", C(4, *QKV, group=128), 64, 8, bias=True, J=2),
    ConsumerCase("cons-w4-g72-m40", C(4, 2048, 1023, group=72), 40, 64, res=True, J=2),
    ConsumerCase("cons-w8-m20", C(8, 1024, 1024), 20, 3, alpha=0.5, J=1),
    ConsumerCase("cons-w16-lmhead-m17", C(16, 1024, 4100), 17, 28, act=X.ACT_RELU),
    ConsumerCase("cons-w16-m64-fp16", C(16, 1024, 1290, ft="fp16"), 64, 3, res=True),
    ConsumerCase("cons-tail65", C(4, 1024, 1290), 65, 8, res=True, bias=True),
    ConsumerCase("cons-tail100", C(4, 1024, 1290), 100, 64, alpha=-1.0, bias=True),
    ConsumerCase("cons-tail128-fp16", C(4, 1024, 1290, ft="fp16"), 128, 28, res=True),
    ConsumerCase("cons-split1", C(4, *QKV), 40, 28, env={"B2_GEMM_TC_MAX_SPLIT": "1"}, bias=True),
    ConsumerCase("cons-g128-pair", C(4, 1024, 1000, group=128, pair=True), 20, 3, J=2),
]


# --------------------------------------------------------------------------------------------------- producer -> consumer
@dataclass
class ChainCase:
    """A hand-off producer (o_proj / down_proj shape, W4 per channel, residual, xg_out + sumsq_out) feeding a consumer
    (gate+up pair, qkv, or a W16 lm_head-shaped GEMM) at M rows.  The consumer is restated from the xg and sumsq_out the
    producer wrote: P = the producer's n-groups, hidden = its N."""
    id: str
    prod: X.Case
    cons: X.Case
    M: int
    bias: bool = False
    path: str = "tc"
    env: dict = field(default_factory=dict)
    act: int = X.ACT_NONE
    alpha: float = 1.0
    res: bool = False


def chain_inputs(ch):
    """Producer: one-hot rows (k_m spread over K) into int4 weights (q - 8) / 8 that are zero three times in four, plus a
    residual j / 8, |j| <= 1, so C = res + (q[k_m] - 8) / 8 has at most 5 significant bits; gamma_out in {1, 0.75, 1.5,
    1.25}: xg = C * gamma_out is exact and on a 2^-5 grid, coarse enough for the consumer's exact accumulation.  Consumer:
    gemm_exact weights (and a bias for qkv)."""
    p, c = ch.prod, ch.cons
    r = np.random.default_rng(_seed(ch.id))
    q = np.full((p.K, p.N), 8, np.uint8)
    nz = r.random((p.K, p.N)) < 0.25
    q[nz] = (8 + r.choice([-2, -1, 1, 2], size=int(nz.sum()))).astype(np.uint8)
    wp = X.Weights(q=q, s=np.full((1, p.N), 0.125), z=np.full((1, p.N), 8.0), unit_s=0.125, unit_z=1.0)
    ks = (np.arange(ch.M) * 7919) % p.K
    A = X.onehot_acts(ks, p.K)
    res = r.integers(-1, 2, size=(ch.M, p.N)) / 8.0
    gamma = np.array([1.0, 0.75, 1.5, 1.25])[np.arange(p.N) % 4]
    wt = X.make_weights(c, _seed(ch.id) + 1)
    wt2 = X.make_weights(c, _seed(ch.id) + 2) if c.pair else None
    bias = X.make_vec(c.N, _seed(ch.id) + 3) if ch.bias else None
    return dict(prod=dict(wt=wp, wt2=None, A=A, res=res, bias=None), gamma=gamma, wt=wt, wt2=wt2, bias=bias, res=None)


def chain_consumer(ch):
    """The ConsumerCase the chain's consumer half is restated as."""
    return ConsumerCase(ch.id, ch.cons, ch.M, ch.prod.NG, bias=ch.bias, hidden=ch.prod.N)


CHAIN_CASES = [
    ChainCase("chain-o-gateup-m17", C(4, *O), C(4, *GU, pair=True), 17),
    ChainCase("chain-o-gateup-m64-fp16", C(4, *O, ft="fp16"), C(4, *GU, pair=True, ft="fp16"), 64),
    ChainCase("chain-o-gateup-m100", C(4, *O), C(4, *GU, pair=True), 100),
    ChainCase("chain-down-qkv-m17-fp16", C(4, 18944, 3584, ft="fp16"), C(4, *QKV, ft="fp16"), 17, bias=True),
    ChainCase("chain-down-qkv-m100", C(4, 18944, 3584), C(4, *QKV), 100, bias=True),
    ChainCase("chain-down-lmhead-m64", C(4, 18944, 3584), C(16, 3584, 4100), 64),
    ChainCase("chain-down-lmhead-m100-fp16", C(4, 18944, 3584, ft="fp16"), C(16, 3584, 4100, ft="fp16"), 100),
]
