"""Exact references, kernel restatements and per-element bounds for the decode step's glue kernels (csrc/glue.cu) and the
rotary embedding of the span-cache appends (span_attn.cu, span_attn64.cu).

RMSNorm.  exact = x g / sqrt(mean(x^2) + eps) in fp64 from the stored inputs (eps as the fp32 the kernel receives).  The
kernel squares in fp32 (exact for 16-bit inputs), sums each thread's 8-element chunks (stride 2048) sequentially, then 5
butterfly levels and 8 warp partials; divides by cols, adds eps, takes rsqrtf (2 ulp), and multiplies by inv and gamma.  Its
fp32 result is within eps_rms(cols) |exact| of exact (rms_eps derives it), and one rounding to FT adds half an FT ulp:
    |y - exact| <= ulp_FT(exact) / 2 + eps_rms(cols) |exact|.
Contract: finite inputs with sum(x^2) < 2^127 (the sum of squares must not overflow fp32 before the divide); the large-row
cases go up to 2^125.

Rotary (NeoX rotate-half over the first rotary_dim dims, half = rotary_dim / 2, partner of dim d: d +- half).  The kernels
compute inv = exp2f(-L * (2 f / rotary_dim)) with L = log2f(base) and f = d % half, angle = fl32(pos * inv), sincosf, and
x cos -+ partner sin in fp32, rounded once to FT.  Against that formula evaluated in fp64 at the fp32 angle of the same
inv (rope_formula), per element:
    |y - Y| <= ulp_FT(|Y| + D) / 2 + D,   D = (|x| + |partner|) (dang + 2^-22)
where dang = pos inv (2^-22 + ln2 |z| 2^-23) + ulp32(angle) for f > 0 (exp2f's 2 ulp and a 1-ulp host log2f, through
z = -L 2f/rotary_dim), 0 for f = 0 (exp2f(0) = 1 exactly); 2^-22 holds sincosf's 2 ulp and the fp32 products.  Against fp64
NeoX (theta = base^(-2f/rotary_dim) exactly) the angle error is at most pos theta (2^-22 + 2^-24 + 1.5 ln2 |z| 2^-23) <=
pos 2^-21 (theta ln(1/theta) <= 1/e), so
    |y - Y64| <= ulp_FT(|Y64| + D64) / 2 + D64,   D64 = (|x| + |partner|) (2^-22 + pos 2^-21).

Argmax.  The order is torch.argmax's: NaN above every number, the lowest index among equal values or among NaNs.  The
reference is np.argmax of the fp32-widened row (which follows that order) plus id_offset; ids and vals_out are exact.
argmax_blocked restates the kernel's reduction (1024 threads striding the row, two butterfly levels of 32) with a
comparison rule, so the CPU tests can show the rule, not just the answer."""
import math

import numpy as np
import torch

U32 = 2.0 ** -24  # unit roundoff of fp32
FTS = {"bf16": torch.bfloat16, "fp16": torch.float16}
_FMT = {torch.bfloat16: (8, -126), torch.float16: (11, -14)}  # (significand bits, least normal exponent)


def ulp(v, dt):
    """ulp of the FT dt at |v| (the subnormal spacing below the normal range)"""
    p, emin = _FMT[dt]
    e = np.floor(np.log2(np.maximum(np.abs(np.asarray(v, np.float64)), 2.0 ** emin)))
    return 2.0 ** (e - (p - 1))


def rn(v, dt):
    """round fp64 values to the nearest dt value, ties to even (one rounding), as fp64; overflow is not handled (no
    reference here leaves the FT range)"""
    v = np.asarray(v, np.float64)
    q = ulp(v, dt)
    return np.round(v / q) * q


def to_ft(x, dt):
    """fp32 values -> dt tensor (torch rounds to nearest even)"""
    return torch.from_numpy(np.ascontiguousarray(x, np.float32)).to(dt)


def ft_values(x, dt):
    """values of x after one rounding to dt, as fp32"""
    return to_ft(x, dt).float().numpy()


# ---------------------------------------------------------------- RMSNorm
RMS_COLS = [8, 56, 896, 2040, 2048, 2056, 3584, 4096, 8192, 18944]
RMS_ROWS = [1, 3, 64, 130]
RMS_EPS = [1e-6, 1e-5]
RMS_KINDS = ["random", "constant", "dominant", "zero", "tiny", "large"]
MISMATCH_PER = 256  # at most ceil(n / 256) elements of a launch may differ from rn_FT(exact)


def rms_depth(cols):
    """additions a square passes through on its way into the row sum: the thread's chunks, 5 butterfly levels, 7 warp
    partials"""
    return 8 * ((cols + 2047) // 2048) + 12


def rms_eps(cols):
    """relative error of the kernel's fp32 result: the sum (depth d, all terms >= 0) and the divide give (d + 1) u on the
    mean, + eps one more u, the square root halves that; rsqrtf adds 2 ulp (4 u), the two products 2 u; 1.01 covers the
    second-order terms"""
    d = rms_depth(cols)
    return 1.01 * ((d + 2) / 2 + 4 + 2) * U32


def rms_exact(x, g, eps):
    x64, g64 = np.asarray(x, np.float64), np.asarray(g, np.float64)
    ms = np.mean(x64 * x64, axis=-1, keepdims=True)
    return x64 * g64 / np.sqrt(ms + float(np.float32(eps)))


def rms_kernel32(x, g, eps, variant=None):
    """the kernel's fp32 formula in numpy with its summation order (rsqrt correctly rounded).  variant: 'eps_outside'
    (x g / (sqrt(mean) + eps)) or 'sum' (sum of squares instead of the mean) are the wrong formulas the bound must reject"""
    x = np.asarray(x, np.float32)
    rows, cols = x.shape
    nchunk = (cols + 2047) // 2048
    xp = np.zeros((rows, nchunk * 2048), np.float32)
    xp[:, :cols] = x
    part = np.zeros((rows, 256), np.float32)
    blk = xp.reshape(rows, nchunk, 256, 8)
    for c in range(nchunk):
        for j in range(8):
            part = part + blk[:, c, :, j] * blk[:, c, :, j]  # fp32: the square is exact, one rounding per add
    w = part.reshape(rows, 8, 32)
    for o in (16, 8, 4, 2, 1):
        w = w + w[:, :, np.arange(32) ^ o]
    tot = np.zeros(rows, np.float32)
    for i in range(8):
        tot = tot + w[:, i, 0]
    e32 = np.float32(eps)
    if variant == "sum":
        ms = tot
    else:
        ms = tot / np.float32(cols)
    if variant == "eps_outside":
        inv = np.float32(1.0) / (np.sqrt(ms.astype(np.float64)) + np.float64(e32)).astype(np.float32)
    else:
        inv = (1.0 / np.sqrt((ms + e32).astype(np.float64))).astype(np.float32)
    return (x * inv[:, None]) * np.asarray(g, np.float32)


def rms_rows(kind, rows, cols, dt, rng):
    """fp32 values exactly representable in dt"""
    if kind == "random":
        x = rng.standard_normal((rows, cols)) * 2.0 ** rng.uniform(-4, 4, (rows, 1))
    elif kind == "constant":
        x = np.ones((rows, cols)) * rng.uniform(-3, 3, (rows, 1))
    elif kind == "dominant":
        x = rng.standard_normal((rows, cols)) * 1e-3
        x[np.arange(rows), rng.integers(0, cols, rows)] = 1000.0 * rng.choice([-1, 1], rows)
    elif kind == "zero":
        x = np.zeros((rows, cols))
    elif kind == "tiny":  # mean(x^2) ~ 1e-10: eps dominates the root by 10^4
        x = rng.standard_normal((rows, cols)) * 1e-5
    elif kind == "large":
        if dt == torch.float16:  # the whole fp16 range: sum(x^2) <= cols 65504^2 < 2^47
            x = np.clip(rng.standard_normal((rows, cols)) * 30000, -65504, 65504)
        else:  # sum(x^2) about 2^125 (cols * 1.0 * s^2), under the 2^127 contract even with 4-sigma rows
            x = rng.standard_normal((rows, cols)) * math.sqrt(2.0 ** 125 / cols)
    else:
        raise ValueError(kind)
    return ft_values(x, dt)


def rms_gamma(cols, dt, rng):
    return ft_values(rng.uniform(-2, 2, cols), dt)


def rms_batch(rows, cols, dt, seed):
    """rows of every kind (row r has kind r % 6) and gamma"""
    rng = np.random.default_rng(seed)
    x = np.concatenate([rms_rows(RMS_KINDS[r % len(RMS_KINDS)], 1, cols, dt, rng) for r in range(rows)])
    return x, rms_gamma(cols, dt, rng)


def rms_check(y, x, g, eps, dt):
    """(worst |y - exact| / bound, elements != rn_FT(exact), elements); zero rows must give exact zeros"""
    ex = rms_exact(x, g, eps)
    y = np.asarray(y, np.float64)
    bound = ulp(ex, dt) / 2 + rms_eps(x.shape[-1]) * np.abs(ex)
    zero = ~np.any(np.asarray(x) != 0, axis=-1)
    if zero.any() and np.any(y[zero] != 0):
        return math.inf, y.size, y.size
    ratio = np.abs(y - ex) / bound
    return float(ratio.max()), int(np.count_nonzero(y != rn(ex, dt))), y.size


def rms_allowed_mismatches(n):
    return -(-n // MISMATCH_PER)


# ---------------------------------------------------------------- rotary
ROPE_POS = [0, 1, 15, 16, 127, 128, 4095, 32767, 131071]
ROPE_BASES = [1e4, 5e5, 1e6]


def rope_tables(base, rotary_dim):
    """per rotated dim d < rotary_dim: (f, z, inv) of the kernels' fp32 formula"""
    half = rotary_dim // 2
    f = np.arange(rotary_dim) % half
    L = np.float32(np.log2(np.float64(np.float32(base))))
    t = (np.float32(2.0) * f.astype(np.float32)) / np.float32(rotary_dim)   # exact: rotary_dim is a power of two
    z = (-L * t).astype(np.float32)
    inv = np.exp2(z.astype(np.float64)).astype(np.float32)
    return f, z, inv


def _partner(x, rotary_dim, wrong=None):
    """rotate-half partner (-x[d + half] for d < half, x[d - half] above), on the last axis; wrong='partner' takes the
    neighbouring dim instead"""
    half = rotary_dim // 2
    a = x[..., :rotary_dim]
    if wrong == "partner":
        return np.concatenate([-a[..., 1:half + 1], a[..., half - 1:rotary_dim - 1]], -1)
    return np.concatenate([-a[..., half:], a[..., :half]], -1)


def rope_formula(x, pos, base, rotary_dim, wrong=None):
    """The kernels' formula at the fp32 angle, evaluated in fp64 (Y), and the per-element slack D of the bound.
    x [..., head] fp32 (rows of one position each, pos broadcast over the leading axes as [..., 1]); dims >= rotary_dim
    are returned unchanged (Y = x, D = 0).  wrong: 'partner', 'sign' or 'pos' (position + 1), the variants the bound
    rejects."""
    x = np.asarray(x, np.float32)
    pos = np.asarray(pos)[..., None]
    if wrong == "pos":
        pos = pos + 1
    f, z, inv = rope_tables(base, rotary_dim)
    ang = (pos.astype(np.float32) * inv).astype(np.float32)
    a = x[..., :rotary_dim].astype(np.float64)
    o = _partner(x, rotary_dim, wrong).astype(np.float64)
    if wrong == "sign":
        o = -o
    ang64 = ang.astype(np.float64)
    Y = x.astype(np.float64).copy()
    Y[..., :rotary_dim] = a * np.cos(ang64) + o * np.sin(ang64)
    dang = np.where(f > 0, pos * inv.astype(np.float64) * (2.0 ** -22 + math.log(2) * np.abs(z) * 2.0 ** -23)
                    + 2.0 ** (np.floor(np.log2(np.maximum(ang64, 2.0 ** -126))) - 23), 0.0)
    D = np.zeros_like(Y)
    D[..., :rotary_dim] = (np.abs(a) + np.abs(o)) * (dang + 2.0 ** -22)
    return Y, D


def rope_neox64(x, pos, base, rotary_dim):
    """fp64 NeoX (theta = base^(-2f/rotary_dim)) and the position-only slack D64 = (|x| + |partner|)(2^-22 + pos 2^-21)"""
    x = np.asarray(x, np.float64)
    pos = np.asarray(pos, np.float64)[..., None]
    half = rotary_dim // 2
    th = np.float64(base) ** (-(np.arange(rotary_dim) % half) * 2.0 / rotary_dim)
    a, o = x[..., :rotary_dim], _partner(x, rotary_dim)
    Y = x.copy()
    Y[..., :rotary_dim] = a * np.cos(pos * th) + o * np.sin(pos * th)
    D = np.zeros_like(Y)
    D[..., :rotary_dim] = (np.abs(a) + np.abs(o)) * (2.0 ** -22 + pos * 2.0 ** -21)
    return Y, D


def rope_ratio(y, Y, D, dt):
    """|y - Y| / (ulp_FT(|Y| + D) / 2 + D) per element"""
    y = np.asarray(y, np.float64)
    return np.abs(y - Y) / (ulp(np.abs(Y) + D, dt) / 2 + D)


def rope_kernel32(x, pos, base, rotary_dim, dt):
    """the kernels' formula in numpy fp32 (sin / cos of the fp32 angle rounded to fp32), rounded once to dt"""
    x = np.asarray(x, np.float32)
    f, z, inv = rope_tables(base, rotary_dim)
    ang = (np.asarray(pos)[..., None].astype(np.float32) * inv).astype(np.float32)
    cs, sn = np.cos(ang.astype(np.float64)).astype(np.float32), np.sin(ang.astype(np.float64)).astype(np.float32)
    y = x.copy()
    y[..., :rotary_dim] = x[..., :rotary_dim] * cs + _partner(x, rotary_dim) * sn
    return ft_values(y, dt)


# ---------------------------------------------------------------- argmax
ARGMAX_N = [1, 31, 1023, 1024, 1025, 128256, 151936, 152064]
ARGMAX_BATCH = [1, 64, 65]
ARGMAX_KINDS = ["random", "tie_stride", "tie_lanes", "tie_warps", "tie_final", "first_last", "equal", "neg_inf", "pos_inf",
                "nan_all", "nan_some"]
TIE_PLANTS = {  # index pairs that tie at the row maximum, by the reduction step that decides them
    "tie_stride": (7, 7 + 1024),   # one thread's sequential loop
    "tie_lanes": (8, 9),           # the first butterfly (lanes of one warp)
    "tie_warps": (3, 3 + 32),      # neighbouring warps, decided in the final warp reduction ...
    "tie_final": (40, 31 * 32 + 2),  # ... and across its widest step (warp 1 vs warp 31)
}
PAD_PLANTS = (np.float32(3e38), np.inf, np.nan)  # in the columns n .. ld - 1, which must be ignored


def argmax_row(kind, n, rng):
    """one fp32 row of n values (representable in bf16 and fp16 alike: multiples of 2^-6 in [-4, 4], specials)"""
    x = np.round(rng.uniform(-4, 4, n) * 64) / 64
    if kind in TIE_PLANTS:
        for i in TIE_PLANTS[kind]:
            x[i % n] = 8.0
    elif kind == "first_last":
        x[0] = x[n - 1] = 8.0
    elif kind == "equal":
        x[:] = 1.5
    elif kind == "neg_inf":
        x[:] = -np.inf
    elif kind == "pos_inf":
        x[rng.integers(0, n, 3)] = np.inf
        x[n // 2] = np.inf
    elif kind == "nan_all":
        x[:] = np.nan
    elif kind == "nan_some":
        x[rng.integers(0, n, 2)] = np.inf
        x[rng.integers(0, n, 3)] = np.nan
    elif kind != "random":
        raise ValueError(kind)
    return x.astype(np.float32)


def argmax_batch(n, batch, pad, seed):
    """[batch, n + pad] fp32: row r of kind r % 11 in the first n columns, PAD_PLANTS cycled in the padding"""
    rng = np.random.default_rng(seed)
    x = np.empty((batch, n + pad), np.float32)
    for r in range(batch):
        x[r, :n] = argmax_row(ARGMAX_KINDS[r % len(ARGMAX_KINDS)], n, rng)
        for j in range(pad):
            x[r, n + j] = PAD_PLANTS[(r + j) % len(PAD_PLANTS)]
    return x


def argmax_ref(x, n, id_offset=0):
    """(ids, vals): np.argmax of the first n columns (the first NaN if any, else the lowest index of the maximum)"""
    x = np.asarray(x, np.float32)[:, :n]
    i = np.argmax(x, axis=1)
    return i.astype(np.int64) + id_offset, x[np.arange(x.shape[0]), i]


def beats(v, i, best, bi):
    """the kernels' order (argmax_beats): NaN above every number; lower index among equals / NaNs"""
    vn, bn = np.isnan(v), np.isnan(best)
    return np.where(vn != bn, vn, (~vn & (v > best)) | ((vn | (v == best)) & (i < bi)))


def beats_before_nan_fix(v, i, best, bi):
    """the rule before NaN was ordered: every comparison with NaN is false"""
    return (v > best) | ((v == best) & (i < bi))


def beats_highest_tie(v, i, best, bi):
    """a wrong rule: ties resolved to the highest index"""
    return (v > best) | ((v == best) & ((i > bi) | (bi == 0x7FFFFFFF)))


def argmax_blocked(row, rule=beats):
    """the kernel's reduction of one row under `rule`: 1024 threads stride the row from (-inf, INT_MAX), butterfly over
    each warp's 32 lanes, then over the 32 warp winners; returns lane 0's (index, value)"""
    row = np.asarray(row, np.float32)
    n = row.shape[0]
    t = np.arange(1024)
    best = np.full(1024, -np.inf, np.float32)
    bi = np.full(1024, 0x7FFFFFFF, np.int64)
    for k in range(0, n, 1024):
        i = t + k
        ok = i < n
        v = row[np.minimum(i, n - 1)]
        m = ok & rule(v, i, best, bi)
        best, bi = np.where(m, v, best), np.where(m, i, bi)

    def butterfly(best, bi):
        best, bi = best.reshape(-1, 32), bi.reshape(-1, 32)
        for o in (16, 8, 4, 2, 1):
            ov, oi = best[:, np.arange(32) ^ o], bi[:, np.arange(32) ^ o]
            m = rule(ov, oi, best, bi)
            best, bi = np.where(m, ov, best), np.where(m, oi, bi)
        return best[:, 0], bi[:, 0]
    best, bi = butterfly(best, bi)
    best, bi = butterfly(best, bi)
    return int(bi[0]), best[0]


def merge_ref(vals, ids, rule=beats):
    """b2_argmax_merge restated: [nranks, batch] pairs, the winner under rule (index = rank, so ties keep the lower rank)"""
    vals, ids = np.asarray(vals, np.float32), np.asarray(ids)
    best, bid = vals[0].copy(), ids[0].copy()
    for r in range(1, vals.shape[0]):
        m = rule(vals[r], 0, best, 0)
        best, bid = np.where(m, vals[r], best), np.where(m, ids[r], bid)
    return bid


def shard_bounds(n, tp):
    """contiguous vocab shards [s, e) of a tp-way split (the last may be shorter)"""
    per = -(-n // tp)
    return [(r * per, min(n, (r + 1) * per)) for r in range(tp)]


def tp_row(kind, n, tp, rng):
    """rows whose winner the vocab split makes hard: on a shard's first / last id, tied across shards, NaN in two shards"""
    x = np.round(rng.uniform(-4, 4, n) * 64) / 64
    b = shard_bounds(n, tp)
    if kind == "edge_first":
        x[b[-1][0]] = 8.0
    elif kind == "edge_last":
        x[b[0][1] - 1] = 8.0
    elif kind == "tie_shards":  # the same maximum in the last id of shard 0 and the first of the last shard
        x[b[0][1] - 1] = x[b[-1][0]] = 8.0
    elif kind == "tie_all_shards":
        for s, _ in b:
            x[s] = 8.0
    elif kind == "nan_shards":
        x[b[-1][0] + 3] = x[b[1][0] + 5] = np.nan
        x[b[0][0]] = np.inf
    elif kind == "neg_inf":
        x[:] = -np.inf
    elif kind != "random":
        raise ValueError(kind)
    return x.astype(np.float32)


TP_KINDS = ["random", "edge_first", "edge_last", "tie_shards", "tie_all_shards", "nan_shards", "neg_inf"]


# ---------------------------------------------------------------- binary / embedding
BINARY_N = [1, 7, 8, 9, 2047, 2048, 2049, 64 * 3584 + 3]
EMBED_HIDDEN = [8, 896, 3584, 8192]


def binary_ref(a, b, op_add, dt):
    """the contract: the fp32 op, one rounding to dt (torch rounds to nearest even and overflows to +-inf)"""
    a, b = torch.as_tensor(a).float(), torch.as_tensor(b).float()
    return (a + b if op_add else a * b).to(dt)
