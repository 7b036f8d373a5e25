"""Exact references, a restatement and per-element bounds for the decode step's log-probabilities (csrc/logprobs.cu:
b2_logprobs, b2_logprobs_shard, b2_logprobs_merge).

Definitions.  For a row x of n values (FT widened to fp32 exactly), m = the maximum under argmax order, and
    lp_i = (x_i - m) - logf(s),   s = sum_i expf(x_i - m)   (all in fp32).
The reference is log_softmax of the widened row in fp64 (torch.log_softmax(x.double())); top_ids is the first n_top entries
in argmax order (glue_ref.beats: NaN first, then descending value, then the lower index), padded with id -1 / lp -inf past n.
Rows whose maximum is not finite (a NaN, a +inf, all -inf) follow torch exactly: every lp of the row is NaN.

The bound (lp_bound), from the kernel's order of operations.  u = 2^-24.  A term t_i = exp(x_i - m) reaches s through the
rounding of x_i - m (a factor exp(u |x_i - m|) on the term), expf's 2 ulp (1 + 2^-22), and d = ceil(n / (1024 C)) + 8 + C
rounded additions (each thread's sequential sum of at most ceil(n / (1024 C)) terms from 0, then 5 + 5 butterfly levels,
then the C CTA partials in order; C = 8 CTAs per row above n = 32768, else 1): all terms are positive, so
    |s^ - s| <= sum_i t_i ((1 + 2^-22) exp(u |x_i - m|) (1 + u)^d - 1) + n 2^-148 (1 + u)^d  =:  e_s s
(2^-148: expf's 2 ulp on a subnormal result).  logf(s^) then differs from L = log s by at most -log(1 - e_s) plus its own
ulp, 2^-23 |log s^|:
    dL = -log(1 - e_s) + 2^-23 (|L| - log(1 - e_s)).
lp_i = fl(fl(x_i - m) - logf(s^)) adds u |x_i - m| and one rounding of the result:
    |lp_i - exact_i| <= (1 + u)(u |x_i - m| + dL) + u |exact_i|.
A result whose magnitude reaches the fp32 overflow threshold is -inf (only bf16 rows spanning +-3e38 get there).

The merge (b2_logprobs_merge over vocab shards q): M = max m_q, S = sum_q fma(s_q, expf(m_q - M), S) in rank order, ranks
with m_q = -inf skipped.  Each rank's s_q carries its own e_s (its own n and d); a rank with m_q != M adds the rounding of
m_q - M and expf's 2 ulp, and with more than one rank every fused multiply-add rounds once ((1 + u)^nranks).  With one rank
m_0 = M, expf(0) = 1 and fma(s, 1, 0) = s exactly, so the merge adds nothing."""
import math

import numpy as np
import torch

U = 2.0 ** -24
EXP_REL = 2.0 ** -22  # expf: 2 ulp
EXP_ABS = 2.0 ** -148  # expf: 2 ulp of the smallest subnormal
FLT_OVF = (2.0 - 2.0 ** -24) * 2.0 ** 127  # fp32 round-to-nearest sends magnitudes from here up to inf
THREADS = 1024   # per CTA
SPLIT_MIN, SPLIT_CTAS = 32768, 8  # rows longer than SPLIT_MIN run on a cluster of SPLIT_CTAS CTAs


def ctas(n):
    return SPLIT_CTAS if n > SPLIT_MIN else 1
N_TOPS = [0, 1, 5, 10]
MAX_TOP = 10


# ---------------------------------------------------------------- references
def lp_exact(x, n):
    """torch.log_softmax of the first n columns of each row in fp64 (fp64 numpy [rows, n])"""
    return torch.log_softmax(torch.from_numpy(np.asarray(x, np.float32)[:, :n].astype(np.float64)), -1).numpy()


def top_order(x, n, n_top):
    """[rows, n_top] int64: the first n_top ids of each row in argmax order, -1 past n"""
    x = np.asarray(x, np.float32)[:, :n]
    out = np.full((x.shape[0], n_top), -1, np.int64)
    idx = np.arange(n)
    for r in range(x.shape[0]):
        nan = np.isnan(x[r])
        key = np.where(nan, 0.0, -x[r].astype(np.float64))
        order = np.lexsort((idx, key, ~nan))  # NaN first (by index), then descending value, then index
        k = min(n, n_top)
        out[r, :k] = order[:k]
    return out


def depth(n):
    """rounded additions on a term's way into s: the thread's ceil(n / (1024 C)) terms summed from 0, 5 + 5 butterfly
    levels, then the C CTA partials added in order (C = ctas(n))"""
    c = ctas(n)
    return -(-n // (THREADS * c)) + 8 + c


def _shard_terms(xq, m):
    """(sum of the terms, relative error e_s of the kernel's s) of one shard against its maximum m (finite)"""
    d64 = xq.astype(np.float64) - m
    t = np.exp(d64)
    fac = (1 + EXP_REL) * np.exp(np.minimum(U * np.abs(d64), 1.0)) * (1 + U) ** depth(xq.size) - 1
    ssum = float(t.sum())
    err = float((t * np.where(t > 0, fac, 0.0)).sum()) + xq.size * EXP_ABS * (1 + U) ** depth(xq.size)
    return ssum, err / ssum


def _max_beats(vals):
    """the maximum under argmax order (NaN above every number)"""
    vals = np.asarray(vals, np.float32)
    return vals[np.isnan(vals)][0] if np.isnan(vals).any() else vals.max()


def lp_bound(x, n, shards=None):
    """(exact [rows, n] fp64, bound [rows, n] fp64).  shards: [(start, end)] of a vocab split (None: the whole row).  Rows
    whose maximum is not finite get bound 0 (they must match torch's NaN / -inf exactly)."""
    x = np.asarray(x, np.float32)[:, :n]
    exact = lp_exact(x, n)
    bound = np.zeros_like(exact)
    shards = shards or [(0, n)]
    for r in range(x.shape[0]):
        M = float(_max_beats(x[r]))
        if not math.isfinite(M):
            continue
        num, den = 0.0, 0.0
        for q, (a, e) in enumerate(shards):
            xq = x[r, a:e]
            mq = float(_max_beats(xq))
            if mq == -math.inf:
                continue
            sq, esq = _shard_terms(xq, mq)
            w = math.exp(mq - M)
            fac = (1 + esq) * ((1 + EXP_REL) * math.exp(min(U * abs(mq - M), 1.0)) if mq != M else 1.0)
            fac *= (1 + U) ** len(shards) if len(shards) > 1 else 1.0
            num += sq * w * (fac - 1) + (sq * EXP_ABS if mq != M else 0.0)
            den += sq * w
        e_s = num / den
        L = math.log(den)
        dL = -math.log1p(-e_s) + 2.0 ** -23 * (abs(L) - math.log1p(-e_s))
        dx = np.abs(x[r].astype(np.float64) - M)
        with np.errstate(invalid="ignore"):
            bound[r] = (1 + U) * (U * dx + dL) + U * np.abs(exact[r])
        bound[r][~np.isfinite(bound[r])] = 0.0  # -inf entries: exact -inf, matched exactly
    return exact, bound


def lp_ratio(got, exact, bound):
    """worst |got - exact| / bound over the elements (inf on any mismatch of a non-finite value).  Where the exact value is
    not finite the result must equal it (NaN for NaN); where it is finite, got may be -inf / +inf only if |exact| + bound
    reaches the fp32 overflow threshold."""
    got = np.asarray(got, np.float64)
    exact = np.asarray(exact, np.float64)
    bound = np.asarray(bound, np.float64)
    fin = np.isfinite(exact)
    nonfin_ok = np.where(np.isnan(exact), np.isnan(got), got == exact)
    if not np.all(nonfin_ok[~fin]):
        return math.inf
    ovf = fin & np.isinf(got)
    with np.errstate(invalid="ignore"):
        reach = np.abs(exact) + bound >= FLT_OVF
    if np.any(ovf & (~reach | (np.sign(got) != np.sign(exact)))):
        return math.inf
    ok = fin & ~ovf
    if not ok.any():
        return 0.0
    diff = np.abs(got[ok] - exact[ok])
    if np.any(np.isnan(diff)):
        return math.inf
    b = bound[ok]
    if np.any((b == 0) & (diff > 0)):
        return math.inf
    return float(np.max(np.where(b > 0, diff / np.where(b > 0, b, 1.0), 0.0)))


def gather(vals, ids):
    """vals [rows, n] at ids [rows, k] (id -1: -inf)"""
    ids = np.asarray(ids)
    out = np.take_along_axis(np.asarray(vals, np.float64), np.maximum(ids, 0), 1)
    return np.where(ids >= 0, out, -np.inf)


# ---------------------------------------------------------------- restatement of the kernel (fp32 in numpy)
def kernel_row32(xq, id_offset=0, n_top=MAX_TOP, tok=None, variant=None):
    """The shard record of one row slice, restated: (m, s, tok_logit, tok_where, vals [K], ids [K]) with the kernel's fp32
    arithmetic and summation order (expf and logf correctly rounded here).  variant 'sum_bf16' accumulates each thread's
    terms in bf16 (a wrong kernel the bound must reject)."""
    xq = np.asarray(xq, np.float32)
    n = xq.size
    K = max(n_top, 1)
    order = top_order(xq[None], n, K)[0]
    vals = np.array([xq[i] if i >= 0 else -np.inf for i in order], np.float32)
    ids = np.array([i + id_offset if i >= 0 else 0x7FFFFFFF for i in order], np.int64)
    m = vals[0]
    nc = ctas(n)
    T = THREADS * nc  # thread g = CTA * 1024 + warp * 32 + lane takes the elements g + T j
    c = -(-n // T)
    xp = np.full(c * T, -np.inf, np.float32)
    xp[:n] = xq
    with np.errstate(invalid="ignore", over="ignore"):
        d = (xp - m).astype(np.float32)
        t = np.exp(d.astype(np.float64)).astype(np.float32)
    t[n:] = 0.0
    t = t.reshape(c, T)
    part = np.zeros(T, np.float32)
    for k in range(c):
        part = (part + t[k]).astype(np.float32)
        if variant == "sum_bf16":
            part = torch.from_numpy(part).to(torch.bfloat16).float().numpy()
    w = part.reshape(nc, 32, 32)
    for o in (16, 8, 4, 2, 1):
        w = (w + w[:, :, np.arange(32) ^ o]).astype(np.float32)
    w = w[:, :, 0].copy()
    for o in (16, 8, 4, 2, 1):
        w = (w + w[:, np.arange(32) ^ o]).astype(np.float32)
    s = w[0, 0]
    for q in range(1, nc):  # CTA 0 adds the CTA partials in order
        s = np.float32(s + w[q, 0])
    where, tl = -1, np.float32(np.nan)
    if tok is not None:
        tq = tok - id_offset
        where = int(0 <= tq < n)
        if where:
            tl = xq[tq]
    return (np.float32(m), np.float32(s), tl, where, vals, ids)


def merge32(recs, n_top, variant=None):
    """lp_finish restated over the records of the ranks: (ids_out, tok_lp, top_ids [n_top], top_lp [n_top]).  variant
    'ft_lp' rounds the logprobs to bf16 (the reference's FT logprobs), which the bound must reject."""
    ms = np.array([r[0] for r in recs], np.float32)
    M = _max_beats(ms)
    S = np.float32(0.0)
    with np.errstate(invalid="ignore", over="ignore"):
        for (m, s, *_rest) in recs:
            if m != -np.inf:
                e = np.float32(np.exp(np.float64(np.float32(m - M))))
                S = np.float32(np.float64(s) * np.float64(e) + np.float64(S))  # fma: one rounding
        ls = np.float32(np.log(np.float64(S))) if S > 0 else (np.float32(-np.inf) if S == 0 else np.float32(np.nan))
    cv = np.concatenate([r[4] for r in recs])
    ci = np.concatenate([r[5] for r in recs])
    K = max(n_top, 1)
    nan = np.isnan(cv)
    key = np.where(nan, 0.0, -cv.astype(np.float64))
    order = np.lexsort((ci, key, ~nan))[:K]
    tv, ti = cv[order], ci[order]

    def lp(v):
        with np.errstate(invalid="ignore", over="ignore"):
            r = np.float32(np.float32(v - M) - ls)
        if variant == "ft_lp":
            r = np.float32(torch.tensor(float(r)).to(torch.bfloat16).float().item())
        return r
    top_ids = np.array([i if i != 0x7FFFFFFF else -1 for i in ti[:n_top]], np.int64)
    top_lp = np.array([lp(v) if i != 0x7FFFFFFF else -np.inf for v, i in zip(tv[:n_top], ti[:n_top])], np.float32)
    if any(r[3] < 0 for r in recs):
        tok = tv[0]
    else:
        found = [r[2] for r in recs if r[3] > 0]
        tok = found[0] if found else np.float32(np.nan)
    return int(ti[0]), lp(tok), top_ids, top_lp


def restated(x, n, n_top, tok_ids=None, shards=None, variant=None):
    """the kernel (shards None) or shard kernels + merge restated over the rows of x: (ids [rows], tok_lp [rows], top_ids
    [rows, n_top], top_lp [rows, n_top])"""
    x = np.asarray(x, np.float32)[:, :n]
    shards = shards or [(0, n)]
    out = []
    for r in range(x.shape[0]):
        tok = None if tok_ids is None else int(tok_ids[r])
        recs = [kernel_row32(x[r, a:e], a, n_top, tok, variant) for a, e in shards]
        out.append(merge32(recs, n_top, variant))
    ids = np.array([o[0] for o in out], np.int64)
    tlp = np.array([o[1] for o in out], np.float32)
    tids = np.stack([o[2] for o in out]) if n_top else np.zeros((x.shape[0], 0), np.int64)
    tlps = np.stack([o[3] for o in out]) if n_top else np.zeros((x.shape[0], 0), np.float32)
    return ids, tlp, tids, tlps


# ---------------------------------------------------------------- rows
LP_KINDS = ["tie_nth", "extreme", "underflow"]


def lp_row(kind, n, dt, rng):
    """the three row kinds beyond glue_ref.ARGMAX_KINDS (fp32 values exact in dt):
    tie_nth: four distinct leaders, then 24 entries equal to the 5th value spread over threads and warps (the lowest-index
      rule past the top-1);  extreme: the FT range's ends (bf16 +-3e38, fp16 +-65504) among random values;  underflow: a
      maximum of 0 and a tail 90 .. 110 below it (expf of the tail is subnormal or 0)."""
    x = np.round(rng.uniform(-4, 4, n) * 64) / 64
    if kind == "tie_nth":
        lead = [12.0, 11.0, 10.5, 10.0]
        pos = rng.permutation(n)
        for j, v in enumerate(lead[:n]):
            x[pos[j]] = v
        x[pos[len(lead):len(lead) + 24]] = 9.0
    elif kind == "extreme":
        big = 3e38 if dt == torch.bfloat16 else 65504.0
        k = min(n, 4)
        pos = rng.permutation(n)[:k]
        x[pos] = big * np.array([1, -1, 1, -1][:k])
    elif kind == "underflow":
        x = -rng.uniform(90, 110, n)
        x[rng.integers(0, n)] = 0.0
    else:
        raise ValueError(kind)
    return torch.from_numpy(x.astype(np.float32)).to(dt).float().numpy()
