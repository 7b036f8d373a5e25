"""CPU restatement of b2_sample (include/b200spark.h), in Python integers and numpy.

Philox4x32-10 (Random123's constants), the row order (value descending, the lower id first, -0 equal to +0), the integer
weights, top-k, top-p and the draw.  Weights come in two forms: "exact" rows, on which every fl32((x - m) c) is an integer
j <= 0 and ex2.approx returns 2^j exactly, so the restatement predicts every id; and "fp64" rows (realistic logits), whose
weights 2^((x - m) c) are taken in fp64, with the ambiguity rule of `draw_margins`.  On a flat row (N(0, 1) logits at
t = 1 over 152064 columns) a single weight is about 2^-17 of the sum, below the worst-case error of a running sum, so a
few per cent of such rows are ambiguous; rows whose mass sits in few tokens are almost never.

`variant` restates one wrong kernel each (MUTATIONS); the CPU suite shows that every one of them changes a drawn id."""
import numpy as np

import glue_ref as G

LOG2E_F32 = np.frombuffer(np.uint32(0x3FB8AA3B).tobytes(), np.float32)[0]
M0, M1, W0, W1 = 0xD2511F53, 0xCD9E8D57, 0x9E3779B9, 0xBB67AE85
MASK32 = 0xFFFFFFFF
TWO40 = 1 << 40
P24 = 1 << 24
# ex2.approx.ftz.f32: maximum relative error 2^-22 (PTX ISA); taken twice that here
EX2_REL = 2.0 ** -21

MUTATIONS = ["tie_high", "neg_zero_below", "top_p_gt", "draw_sk", "top_k_plus1", "row_in_counter", "r1", "temp_mul"]


def philox(ctr, key):
    """Philox4x32-10 of counter (c0, c1, c2, c3) and key (k0, k1); numpy uint64 arrays or ints, element-wise"""
    c = [np.asarray(v, np.uint64) for v in ctr]
    k0, k1 = np.asarray(key[0], np.uint64), np.asarray(key[1], np.uint64)
    m32 = np.uint64(MASK32)
    for rnd in range(10):
        if rnd:
            k0, k1 = (k0 + np.uint64(W0)) & m32, (k1 + np.uint64(W1)) & m32
        p0, p1 = np.uint64(M0) * c[0], np.uint64(M1) * c[2]
        c = [((p1 >> np.uint64(32)) ^ c[1] ^ k0) & m32, p1 & m32, ((p0 >> np.uint64(32)) ^ c[3] ^ k1) & m32, p0 & m32]
    return c


def draw_u24(seed, off, row=0, variant=None):
    """u24 of the draw, for uint64 seeds / offsets (scalars or arrays)"""
    seed, off = np.asarray(seed, np.uint64), np.asarray(off, np.uint64)
    ctr = (off & np.uint64(MASK32), off >> np.uint64(32), np.uint64(row if variant == "row_in_counter" else 0), np.uint64(0))
    r = philox(ctr, (seed & np.uint64(MASK32), seed >> np.uint64(32)))
    return (r[1] if variant == "r1" else r[0]) >> np.uint64(8)


def p24_of(p):
    p = np.float32(p)
    if not p < 1:
        return P24
    return int(min(max(np.rint(np.float64(p * np.float32(P24))), 0), P24))


def order(x, variant=None):
    """ids of the row in the sampling order"""
    ids = np.arange(x.shape[0])
    if variant == "tie_high":
        return np.lexsort((-ids, -x))
    if variant == "neg_zero_below":
        return np.lexsort((ids, np.signbit(x) & (x == 0), -x))
    return np.lexsort((ids, -x))


def weights(x, m, c, form="exact"):
    """int64 weights: 0 at -inf, else rint(2^fl32(fl32(x - m) c) 2^40) (exact in the exact form; fp64 otherwise)"""
    y = ((x - np.float32(m)).astype(np.float32) * np.float32(c)).astype(np.float32).astype(np.float64)
    if form == "exact":
        assert np.all((y == np.floor(y)) | np.isneginf(x)), "not an exact row"
    with np.errstate(over="ignore", invalid="ignore"):
        w = np.rint(np.exp2(np.minimum(y, 0.0)) * TWO40)
    w = np.where(np.isneginf(x) | (np.exp2(np.minimum(y, 0.0)) < 2.0 ** -126), 0.0, w)
    return w.astype(np.int64)


def params(t, k, p, n, variant=None):
    """(greedy?, c, k, p24) of a row whose maximum is finite"""
    t = np.float32(t)
    with np.errstate(over="ignore", divide="ignore", invalid="ignore"):
        c = np.float32(LOG2E_F32 * t) if variant == "temp_mul" else np.float32(LOG2E_F32 / t)
    greedy = not (t > 0) or not np.isfinite(c)
    kk = n if (k <= 0 or k > n) else int(k)
    return greedy, c, kk, p24_of(p)


def row_plan(x, t, k, p, form="exact", variant=None):
    """Everything of a row's draw except the random value: None for a greedy row (its id is argmax), else a dict with the
    order, the weights in the order (int64), S_k, Pt, the nucleus length and S_p."""
    x = np.asarray(x, np.float32)
    n = x.shape[0]
    if np.isnan(x).any() or not np.isfinite(x.max()):
        return None
    greedy, c, kk, p24 = params(t, k, p, n, variant)
    if greedy:
        return None
    m = x.max()
    o = order(x, variant)
    w = weights(x, m, c, form)[o]
    if variant == "top_k_plus1":
        kk = min(kk + 1, n)
    cum = np.cumsum(w[:kk])
    Sk = int(cum[-1])
    Pt = max(1, (p24 * Sk + P24 - 1) >> 24)
    npl = int(np.searchsorted(cum, Pt, side="right" if variant == "top_p_gt" else "left")) + 1
    npl = min(npl, kk)
    return {"order": o, "w": w, "cum": cum, "Sk": Sk, "Pt": Pt, "np": npl, "Sp": int(cum[npl - 1]), "kk": kk}


def draw(plan, u24, variant=None):
    """drawn ids for one plan and an array of u24 values"""
    S = plan["Sk"] if variant == "draw_sk" else plan["Sp"]
    u24 = np.asarray(u24, np.uint64).astype(object)
    U = np.array([(int(u) * S) >> 24 for u in np.atleast_1d(u24)], np.int64)
    pos = np.minimum(np.searchsorted(plan["cum"][:plan["np"]], U, side="right"), plan["np"] - 1)
    return plan["order"][pos]


def sample_row(x, t, k, p, seed, off, row=0, form="exact", variant=None):
    """the id b2_sample draws from row x (fp32, the first n columns)"""
    plan = row_plan(x, t, k, p, form, variant)
    if plan is None:
        return int(G.argmax_ref(np.asarray(x, np.float32)[None], x.shape[0])[0][0])
    return int(draw(plan, draw_u24(seed, off, row, variant), variant)[0])


def draw_margins(plan, u24):
    """(unambiguous?) of an fp64-weight row.  A GPU weight differs from the fp64 one by d_i, |d_i| <= W_i EX2_REL + 1
    (ex2.approx's relative error, the two roundings to an integer).  The top-p decision compares the running sum C_j with
    Pt = ceil(p S_k): C_j - p S_k moves by at most (1 - p) sum_{i <= j} |d_i| + p sum_{j < i <= k} |d_i| + 1, and the draw
    compares C_j with U = floor(u S_p) the same way with u = u24 / 2^24 over the nucleus.  A decision is clear when the
    running sums before and at its crossing lie further than that from the threshold; the row is unambiguous when both are."""
    w = plan["w"].astype(np.float64)
    err = w * EX2_REL + 1
    cum = plan["cum"]

    def clear(T, end, f):
        e = np.cumsum(err[:end])
        i = int(np.searchsorted(cum[:end], T, side="left"))
        for q in (i - 1, min(i, end - 1)):
            c, ec = (cum[q], e[q]) if q >= 0 else (0, 0.0)
            if abs(float(c) - float(T)) <= (1 - f) * ec + f * (e[end - 1] - ec) + 2:
                return False
        return True

    if plan["Pt"] < plan["Sk"] and not clear(plan["Pt"], plan["kk"], plan["Pt"] / plan["Sk"]):
        return False  # (Pt = S_k: the nucleus is the kept set on both sides, S_p = S_k)
    U = (int(u24) * plan["Sp"]) >> 24
    return clear(U + 1, plan["np"], int(u24) / P24)


def exact_row(n, j, m, rng, dt, neg_inf=0):
    """a row of n values m - d 2^-j (d small integers, so fl32(x - m) 2^j = -d exactly), representable in dt: weights 2^(40-d)
    or 0; d = 0 appears several times (ties at the maximum, +0 and -0 when m = 0), a few -inf entries"""
    d = np.minimum(rng.geometric(0.15, n) - 1, 50).astype(np.float64)
    d[rng.integers(0, n, max(1, n // 64))] = rng.integers(0, 4, max(1, n // 64))
    x = (np.float64(m) - d * 2.0 ** -j).astype(np.float32)
    if m == 0:
        z = np.flatnonzero(d == 0)
        x[z[::2]] = np.float32(-0.0)
    if neg_inf and n > 1:
        x[rng.integers(0, n, neg_inf)] = -np.inf
        x[np.argmin(d)] = np.float32(m) if m != 0 else np.float32(0.0)
    assert np.array_equal(G.ft_values(x, dt), x, equal_nan=True)
    return x


def exact_temperature(j):
    """fl32(LOG2E_F32 2^-j): c = LOG2E_F32 / t is 2^j exactly"""
    return np.float32(LOG2E_F32 * np.float32(2.0 ** -j))
