"""Exact-arithmetic ("dyadic") inputs for SpanAttention and a restatement of the kernel's arithmetic that predicts every
output bit, plus the error envelope of the honest kernel on realistic data (no absolute floor).

Dyadic cache (written straight into span memory, not through the append kernel):
  * NONE: small integers times a power of two, in bf16 or fp16;
  * I8 / U4: codes u, an integer zero z and a power-of-two scale (value (u - z) s);  FP8: e4m3 codes, zero 0, scale 2^e;
  * Q: small integers.  The query of head h holds 1 in its own reserved dim d_h (the last 16 dims) and small integers
    {-1, 0, 1} elsewhere; a token's K row holds {-1, 0, 1} noise and, in dim d_h, the value that puts head h's score on a
    chosen integer (log2 units) at most D below the row's maximum.  qk_scale is one of the fp32 values that make the
    host's fp32 scale_log2 = qk_scale * 1.4426950408889634f a power of two (exact_qk_scale), and s_k scale_log2 is 1 or 2.
So every score is an integer in log2 units, every probability is 2^-i, and, under the precondition (precondition()),
every sum the kernel forms is an integer multiple of its grid unit below 2^23 units: no rounding happens until the final
normalisation.  The restatement (predict) then repeats that last step in the kernel's own form:
  one piece: rn32(acc / L) (div.rn.f32);  a cross-CTA merge or head 64: rn32(acc * rn32(1 / L));  then one FT store.
exp2f compiles to ex2.approx.f32 (2 ulp documented; exact on integers expected, not assumed): the bound per element is
  1/2 ulp_FT(y) + 2^-21 |y|   (y: the exact value),
and the tests report how many elements differ from the bit prediction (expected 0).  tile_sim() restates the same
arithmetic per piece, tile and warp slice (running max, corr, l, o, cacc, partial slots, merges) so that bugs of the tile
math and of the merges can be applied to it.  Rounding cases (Case.vbits) give V scales 13 significant bits, so that
rn_f16(P s_v 2^E) rounds; their sums are not exact and the bound takes the accumulation term (accum_bound).

Realistic data (envelope()): 1/2 ulp_FT(ref) + u_P sum p|V| / l + score and accumulation terms from the kernel's serial
depth; u_P: the unit roundoff of the probabilities the P V MMA multiplies (bf16 2^-8, fp16 2^-11).  tile_math() restates
the quantized tile math (P' = rn_f16(P s_v 2^E)) to show on the CPU that small V scales need the 2^E of KVTraits::kPExp.
Imports without the native library or a GPU."""
from dataclasses import dataclass

import numpy as np
import torch

import attn_needles as A
import kv_fp8_ref as F8
import tree_ref as TR

NONE, I8, U4, FP8 = A.NONE, A.I8, A.U4, A.FP8
MODES = (NONE, I8, U4, FP8)
NAMES = A.MODE_NAMES
BF16, FP16 = torch.bfloat16, torch.float16
HEAD = 128
R = 16                                       # reserved (steering) dims, one per query row of a kv-group
BIAS = {NONE: 0, I8: 1152, U4: 1024, FP8: 0}  # tile_compute_q: the MMAs multiply BIAS + u
P_EXP = {NONE: 0, I8: 10, U4: 6, FP8: 12}    # KVTraits::kPExp: P' = rn_f16(P * s_v * 2^E)
LOG2E = np.float32(1.4426950408889634)
BUDGET = 2.0 ** 23                           # sums below 2^23 grid units are exact in fp32 whatever the order


def scale_log2(qk_scale):
    """the host's fp32 qk_scale * 1.4426950408889634f"""
    return float(np.float32(np.float32(qk_scale) * LOG2E))


def exact_qk_scale(j):
    """an fp32 qk_scale whose fp32 scale_log2 is exactly 2^-j (searched around 2^-j / log2 e)"""
    x0 = np.float32(2.0 ** -j / 1.4426950408889634)
    for direction in (np.float32(np.inf), np.float32(0)):
        x = x0
        for _ in range(64):
            if scale_log2(x) == 2.0 ** -j:
                return float(x)
            x = np.nextafter(x, direction, dtype=np.float32)
    raise AssertionError("no fp32 qk_scale gives scale_log2 = 2^-%d" % j)


QK_SCALES = {0: 0.6931471824645996, 3: 0.08664339780807495, 4: 0.043321698904037476}


def rn32(x):
    return np.asarray(x, np.float64).astype(np.float32).astype(np.float64)


def rn_f16(x):
    return np.asarray(x, np.float64).astype(np.float32).astype(np.float16).astype(np.float64)


def rn_ft(x, dtype):
    return torch.from_numpy(np.ascontiguousarray(x, np.float32)).to(dtype).double().numpy()


def ulp_ft(y, dtype):
    """the spacing of FT numbers at |y| (fp16: subnormal spacing 2^-24 below 2^-14)"""
    e = np.floor(np.log2(np.maximum(np.abs(y), 2.0 ** -126)))
    return 2.0 ** (e - 7) if dtype == BF16 else 2.0 ** (np.maximum(e, -14) - 10)


# --------------------------------------------------------------------------------------------------------- the cases
@dataclass
class Case:
    name: str
    mode: int
    dtype: object
    span: int
    nH: int
    nG: int
    lens: list                 # new lengths per sequence (tokens the last query row sees)
    form: str = "single"       # "single", "chain" or "tree"
    q_len: int = 1
    parents: list = None       # tree: parents per sequence
    head: int = HEAD
    jexp: int = 3              # scale_log2 = 2^-jexp
    drop: int = 4              # live scores lie in [max - drop - 4, max]
    heavy: float = 0.1         # share of tokens above the floor score (the rest sit at max - drop)
    vexp: int = -1             # V scales 2^vexp or 2^(vexp + 1)
    vbits: int = 0             # > 0: V scales m 2^(vexp - vbits + 1), m odd with vbits bits, so rn_f16(P s_v) rounds
    max_pieces: int = None     # B2_ATTN_MAX_PIECES
    ctas_per_sm: int = None    # B2_ATTN_CTAS_PER_SM
    seed: int = 0

    @property
    def hpg(self):
        return self.nH // self.nG

    @property
    def qk_scale(self):
        return QK_SCALES[self.jexp]

    def rows(self):
        return len(self.lens) * self.q_len

    def visible(self, b, tau):
        """[lens[b]] bool: the tokens query token tau of sequence b sees"""
        L = self.lens[b]
        v = np.zeros(L, bool)
        if self.form == "single":
            v[:] = True
        elif self.form == "chain":
            v[:L - self.q_len + tau + 1] = True
        else:
            v = TR.tree_mask(L, self.parents[b])[tau]
        return v

    def items(self):
        """(item lens, item -> (b, first query token, tokens)) of the kernel's work items (QueryRows)"""
        if self.form == "single":
            return list(self.lens), [(b, 0, 1) for b in range(len(self.lens))]
        tpb = min(self.q_len, 16 // self.hpg)
        nrb = -(-self.q_len // tpb)
        lens, meta = [], []
        for b, L in enumerate(self.lens):
            for rb in range(nrb):
                lens.append(L - self.q_len + min(self.q_len, (rb + 1) * tpb))
                meta.append((b, rb * tpb, min(tpb, self.q_len - rb * tpb)))
        return lens, meta


HPG = [(28, 4), (16, 1), (8, 8), (32, 4), (16, 4)]  # hpg 7, 16, 1, 8, 4
LENS = [1, 15, 16, 63, 64, 65, 127, 128, 129, 2049]


def single_cases():
    out = []
    for mode in MODES:
        for dtype in (BF16, FP16):
            for span in (16, 128):
                nH, nG = HPG[len(out) % len(HPG)]
                lens = LENS[len(out) % 3:] + LENS[:len(out) % 3]
                out.append(Case("%s-%s-s%d-%d/%d" % (NAMES[mode], "bf16" if dtype == BF16 else "fp16", span, nH, nG),
                                  mode, dtype, span, nH, nG, lens, seed=len(out)))
    return out


def step_cases():
    out = []
    shapes = [("chain", 2, None, (16, 4)), ("chain", 5, None, (28, 4)), ("chain", 16, None, (8, 8)),
              ("tree", 8, TR.deepest_last(8), (16, 4)), ("tree", 12, [0, 0, 1, 1, 0, 4, 2, 6, 3, 3, 9, 5], (8, 8))]
    for mode in MODES:
        for form, T, par, (nH, nG) in shapes:
            dtype = FP16 if len(out) % 2 else BF16
            lens = [T, T + 15, 64 + T, 129 + T]
            out.append(Case("%s-%s%d-%s-%d/%d" % (NAMES[mode], form, T, "bf16" if dtype == BF16 else "fp16", nH, nG),
                              mode, dtype, 16 if len(out) % 2 else 128, nH, nG, lens, form=form, q_len=T,
                              parents=[par] * len(lens) if par else None, seed=100 + len(out)))
    return out


def rounding_cases():
    """int8 / uint4 with V scales of 13 significant bits: rn_f16(P s_v 2^E) rounds, so the zero-point term must be built
    from the same rounded P' the MMA multiplies (its error is BIAS times the rounding of P'); the sums are no longer exact
    and the bound takes the accumulation term"""
    out = []
    for mode in (I8, U4):
        out.append(Case("%s-bf16-s16-28/4-vbits13" % NAMES[mode], mode, BF16, 16, 28, 4, [1, 15, 64, 65, 129, 2049], vbits=13,
                        seed=500 + mode))
        out.append(Case("%s-chain5-fp16-16/4-vbits13" % NAMES[mode], mode, FP16, 128, 16, 4, [5, 20, 69, 134], form="chain",
                        q_len=5, vbits=13, seed=510 + mode))
    return out


def merge_cases(grid):
    """the needle suite's merge shapes (B2_ATTN_CTAS_PER_SM=1: grid = the SM count) in every mode"""
    return [Case("merge%d-%s" % (i + 1, NAMES[mode]), mode, BF16, 16, nH, nG, lens, max_pieces=mp, ctas_per_sm=1, seed=200 + i)
            for mode in MODES for i, (lens, nH, nG, mp) in enumerate(A.merge_shape_cases(grid))]


@dataclass
class Data:
    q: np.ndarray              # [rows, nH, head] small integers (fp64)
    kc: list                   # per sequence [W, nG, head]: NONE value / u - z / e4m3 value
    ks: list                   # [W, nG] scale (NONE: 1)
    ku: list                   # [W, nG, head] stored code (int; NONE: the value)
    kz: list                   # [W, nG] zero
    vc: list
    vs: list
    vu: list
    vz: list


_E4M3 = F8.decode(np.arange(256, dtype=np.uint8)).astype(np.float64)
_E4M3_INT = {int(v): c for c, v in enumerate(_E4M3) if np.isfinite(v) and v == int(v) and abs(v) <= 16 and c != 0x80}
_E4M3_V = [c for c, v in enumerate(_E4M3) if np.isfinite(v) and abs(v) <= 32 and v * 8 == int(v * 8)]


def make(case):
    """Dyadic Q, K and V of a case (see the module docstring)."""
    rng = np.random.default_rng(case.seed)
    B, nG, hpg, head, mode = len(case.lens), case.nG, case.hpg, case.head, case.mode
    noise = head - R
    # Q: one base row per head; a multi-token step perturbs one noise dim per query token by +-1
    qb = rng.integers(-1, 2, (B, case.nH, head)).astype(np.float64)
    qb[..., noise:] = 0.0
    for h in range(case.nH):
        qb[:, h, noise + h % hpg] = 1.0
    q = np.repeat(qb[:, None], case.q_len, 1)
    if case.q_len > 1:
        d = rng.integers(0, noise, (B, case.q_len, case.nH))
        s = rng.choice([-1.0, 1.0], (B, case.q_len, case.nH))
        s[:, 0] = 0.0
        np.put_along_axis(q, d[..., None], np.clip(np.take_along_axis(q, d[..., None], -1) + s[..., None], -2, 2), -1)
    q = q.reshape(B * case.q_len, case.nH, head)
    cmax = {NONE: 40, I8: 40, U4: 7, FP8: 16}[mode]
    dens = 0.125 if mode == U4 else 0.25
    kc, ks, ku, kz, vc, vs, vu, vz = ([] for _ in range(8))
    for b, L in enumerate(case.lens):
        ek = rng.integers(0, 2, (L, nG))                      # s_k scale_log2 = 2^ek
        c = (rng.integers(-1, 2, (L, nG, head)) * (rng.random((L, nG, head)) < dens)).astype(np.float64)
        c[..., noise:] = 0.0
        heavy = rng.random((L, nG, hpg)) < case.heavy
        tgt = np.where(heavy, -rng.integers(0, case.drop + 1, (L, nG, hpg)), -case.drop)
        tgt = np.where(ek[..., None] == 1, tgt // 2, tgt)     # raw target; the score is raw * 2^ek
        for g in range(nG):
            qg = qb[b, g * hpg:(g + 1) * hpg]                  # [hpg, head]
            N = c[:, g] @ qg.T                                 # [L, hpg]
            steer = tgt[:, g] - N
            bad = np.abs(steer).max(1) > cmax
            c[bad, g] = 0.0
            steer[bad] = tgt[bad, g]
            c[:, g, noise:noise + hpg] = steer
        # dims noise + hpg .. head - 1 of K: noise nobody's query reads (a wrong d-order picks it up)
        c[..., noise + hpg:] = rng.integers(-1, 2, (L, nG, R - hpg))
        if mode == NONE:
            kv = c * 2.0 ** (case.jexp + ek[..., None])
            kc.append(kv); ks.append(np.ones((L, nG))); ku.append(kv); kz.append(np.zeros((L, nG)))
        else:
            z = rng.integers(-6, 7, (L, nG)).astype(np.float64) if mode == I8 else (
                rng.integers(7, 9, (L, nG)).astype(np.float64) if mode == U4 else np.zeros((L, nG)))
            u = c + z[..., None]
            if mode == FP8:
                u = np.vectorize(_E4M3_INT.__getitem__)(c.astype(int)).astype(np.float64)
            kc.append(c); ks.append(2.0 ** (case.jexp + ek)); ku.append(u); kz.append(z)
        # V
        ev = case.vexp + rng.integers(0, 2, (L, nG))
        if mode == NONE:
            v = rng.integers(-64, 65, (L, nG, head)) * 2.0 ** (ev[..., None] - 4)
            vc.append(v); vs.append(np.ones((L, nG))); vu.append(v); vz.append(np.zeros((L, nG)))
        elif mode == FP8:
            codes = rng.choice(_E4M3_V, (L, nG, head))
            vc.append(_E4M3[codes]); vs.append(2.0 ** ev); vu.append(codes.astype(np.float64)); vz.append(np.zeros((L, nG)))
        else:
            lo, hi = (-128, 128) if mode == I8 else (0, 16)
            u = rng.integers(lo, hi, (L, nG, head)).astype(np.float64)
            z = rng.integers(-4, 5, (L, nG)).astype(np.float64) if mode == I8 else rng.integers(0, 16, (L, nG)).astype(np.float64)
            vc.append(u - z[..., None]); vs.append(2.0 ** ev); vu.append(u); vz.append(z)
        if case.vbits and mode != NONE:
            m = rng.integers(2 ** (case.vbits - 2), 2 ** (case.vbits - 1), (L, nG)) * 2 + 1
            vs[-1] = vs[-1] * m * 2.0 ** (1 - case.vbits)
    return Data(q, kc, ks, ku, kz, vc, vs, vu, vz)


# ---------------------------------------------------------------------------------------------------- span bytes
def span_bytes_of(case, which, data, b):
    """The span byte images of sequence b's K or V rows: [nG][span][ROW] codes, then [nG][span] {f32 zero, f32 scale}"""
    u = (data.ku if which == "k" else data.vu)[b]
    z = (data.kz if which == "k" else data.vz)[b]
    s = (data.ks if which == "k" else data.vs)[b]
    L, nG, head, span, mode = u.shape[0], case.nG, case.head, case.span, case.mode
    out = []
    for si in range(-(-L // span)):
        n = min(span, L - si * span)
        rows = u[si * span:si * span + n].transpose(1, 0, 2)   # [nG, n, head]
        if mode == NONE:
            bits = torch.from_numpy(np.ascontiguousarray(rows, np.float32)).to(case.dtype).view(torch.int16).numpy().view(np.uint8)
            buf = np.zeros((nG, span, head * 2), np.uint8)
            buf[:, :n] = bits.reshape(nG, n, head * 2)
            out.append((buf.reshape(-1), None))
            continue
        if mode == U4:
            codes = rows.astype(np.uint8)
            by = (codes[..., 0::2] | (codes[..., 1::2] << 4)).astype(np.uint8)
        elif mode == I8:
            by = rows.astype(np.int64).astype(np.int8).view(np.uint8)
        else:
            by = rows.astype(np.uint8)
        buf = np.zeros((nG, span, by.shape[-1]), np.uint8)
        buf[:, :n] = by
        prm = np.zeros((nG, span, 2), np.float32)
        prm[:, :n, 0] = z[si * span:si * span + n].T
        prm[:, :n, 1] = s[si * span:si * span + n].T
        out.append((buf.reshape(-1), (prm, n)))
    return out


# -------------------------------------------------------------------------------------------------- arithmetic
def scores(case, data, b, g, rows_q):
    """[nrow, L] exact scores in log2 units of query rows rows_q [nrow, head] against sequence b, kv-head g"""
    sl = 2.0 ** -case.jexp
    K = data.kc[b][:, g] * data.ks[b][:, g, None]
    return (rows_q @ K.T) * sl


def _row_sets(case):
    """(b, tau, h, visible) for every output row"""
    for b in range(len(case.lens)):
        for tau in range(case.q_len):
            vis = case.visible(b, tau)
            for h in range(case.nH):
                yield b, tau, h, vis


def p_prime(mode, P, sv):
    """What the P V MMA multiplies per token, in value units: P (bf16 / fp16 exact for P = 2^-i) or, quantized,
    rn_f16(rn32(P rn32(s_v 2^E))) / 2^E"""
    if mode == NONE:
        return P * sv
    e = 2.0 ** P_EXP[mode]
    return rn_f16(rn32(P * rn32(sv * e))) / e


def exact(case, data):
    """(y, acc, L) per output row: y [rows, nH, head] = acc / L in fp64, acc = sum P' c (P' = p_prime: the probability
    the kernel rounds, times s_v), L = sum P with P = 2^(s - max).  With power-of-two V scales P' = P s_v exactly."""
    B, head = len(case.lens), case.head
    y = np.zeros((B * case.q_len, case.nH, head))
    acc = np.zeros_like(y)
    Ls = np.zeros((B * case.q_len, case.nH))
    for b, tau, h, vis in _row_sets(case):
        g = h // case.hpg
        s = scores(case, data, b, g, data.q[b * case.q_len + tau, h][None])[0]
        s = np.where(vis, s, -np.inf)
        P = np.exp2(s - s.max())
        acc[b * case.q_len + tau, h] = p_prime(case.mode, P, data.vs[b][:, g]) @ data.vc[b][:, g]
        Ls[b * case.q_len + tau, h] = P.sum()
    y = acc / Ls[..., None]
    return y, acc, Ls


def merged_rows(case, grid):
    """[rows, nH] bool: the rows whose (item, kv-head) is split into several pieces (the final step is acc * rcp(L))"""
    out = np.zeros((case.rows(), case.nH), bool)
    if case.head != HEAD:
        return np.ones_like(out)
    lens, meta = case.items()
    dec = A.decompose(lens, case.nG, grid, case.max_pieces)
    for bg in dec.bgs:
        if bg.npieces > 1:
            b, t0, nt = meta[bg.b]
            out[b * case.q_len + t0:b * case.q_len + t0 + nt, bg.g * case.hpg:(bg.g + 1) * case.hpg] = True
    return out


def predict(case, data, grid, ex=None):
    """The output bits the kernel writes when no sum rounds: FT(rn32(acc / L)) or FT(rn32(acc * rn32(1 / L)))"""
    y, acc, Ls = ex if ex is not None else exact(case, data)
    a32, l32 = rn32(acc), rn32(Ls)[..., None]
    if not case.vbits:  # bit-exact only when no sum rounds
        assert np.array_equal(a32, acc) and np.array_equal(l32[..., 0], Ls), "acc / L not fp32 numbers"
    div = rn32(a32.astype(np.float32) / l32.astype(np.float32))
    mul = rn32(a32.astype(np.float32) * (np.float32(1) / l32.astype(np.float32)))
    return rn_ft(np.where(merged_rows(case, grid)[..., None], mul, div), case.dtype)


def bound(case, y):
    return 0.5 * ulp_ft(y, case.dtype) + 2.0 ** -21 * np.abs(y)


def precondition(case, data):
    """Every sum the kernel forms is an integer multiple of its grid unit below 2^23 units.  Checked per output row over
    ALL its visible tokens (the order-free, split-free form: every partial sum of a warp slice, piece or merge is a sub-sum
    of these), for the score sums, l, o = sum P'(BIAS + u), the zero-point term sum P'(BIAS + z), their difference and the
    merged sums.  Returns the worst ratio (sum / unit) / 2^23 (exact when < 1; inf when P' carries 11 significant bits,
    vbits cases, whose sums need more than fp32 holds)."""
    if case.vbits and case.mode != NONE:
        return np.inf
    worst, bias = 0.0, BIAS[case.mode]
    head = case.head
    for b, tau, h, vis in _row_sets(case):
        g = h // case.hpg
        qr = data.q[b * case.q_len + tau, h]
        ku = data.ku[b][vis, g]
        # the raw score sum: integers (or small integers x 2^a for NONE) over head dims
        if case.mode == NONE:
            kv = data.kc[b][vis, g]
            unit = 2.0 ** (case.jexp)
            worst = max(worst, float((np.abs(qr) @ np.abs(kv).T).max()) / unit / BUDGET)
        else:
            k_raw = bias + (ku if case.mode != FP8 else data.kc[b][vis, g])
            worst = max(worst, float((np.abs(qr) @ np.abs(k_raw).T).max()) / BUDGET,
                        float(((bias + np.abs(data.kz[b][vis, g])) * np.abs(qr).sum()).max()) / BUDGET)
        s = scores(case, data, b, g, qr[None])[0][vis]
        assert np.array_equal(s, np.round(s)), "scores not integers in log2 units"
        P = np.exp2(s - s.max())
        worst = max(worst, P.sum() / P.min() / BUDGET)                        # l
        sv = data.vs[b][vis, g] * 2.0 ** P_EXP[case.mode]
        Pq = P * sv
        if case.mode != NONE:
            assert np.all(Pq >= 2.0 ** -14) and np.all(Pq <= 65504), "P' not a normal fp16 number"
        if case.mode == NONE:  # V = integer x 2^(vexp - 4 + {0, 1})
            mag, gran = np.abs(data.vc[b][vis, g]), 2.0 ** (case.vexp - 4)
        elif case.mode == FP8:
            mag, gran = np.abs(data.vc[b][vis, g]), 2.0 ** -3
        else:
            mag, gran = bias + np.maximum(np.abs(data.vu[b][vis, g]), np.abs(data.vz[b][vis, g])[:, None]), 1.0
        unit = Pq.min() * gran
        worst = max(worst, float((Pq @ mag).max()) / unit / BUDGET)
    return worst


def accum_bound(case, data, grid):
    """Cases beyond the exact budget: depth 2^-24 sum P' (BIAS + |u| + |z|) / l per row in value units, depth = the serial
    depth of the split (the tiles of a CTA, the warp merge, the pieces, the MMA's own additions)"""
    lens, _ = case.items()
    dec = A.decompose(lens, case.nG, grid, case.max_pieces)
    depth = dec.Tc + 4 + max(bg.npieces for bg in dec.bgs) + 8
    out = np.zeros((case.rows(), case.nH, case.head))
    bias = BIAS[case.mode]
    for b, tau, h, vis in _row_sets(case):
        g = h // case.hpg
        s = scores(case, data, b, g, data.q[b * case.q_len + tau, h][None])[0][vis]
        P = np.exp2(s - s.max())
        mag = bias + np.abs(data.vu[b][vis, g]) + np.abs(data.vz[b][vis, g])[:, None]
        out[b * case.q_len + tau, h] = depth * 2.0 ** -24 * (p_prime(case.mode, P, data.vs[b][vis, g]) @ mag) / P.sum()
    return out


def case_bound(case, data, grid, y):
    """the per-element bound a GPU case is held to"""
    return bound(case, y) + (accum_bound(case, data, grid) if precondition(case, data) >= 1.0 else 0.0)


# ------------------------------------------------------------------------------------------ tile-level restatement
def tile_sim(case, data, grid, mutant=None):
    """span_attn_kernel's arithmetic restated per piece, tile and warp slice (fp64 sums; exact on dyadic data): online
    softmax with the running max, corr, l, o = sum P'(BIAS + u), the zero-point term cacc = sum P'(BIAS + z), the warp
    merge, the partials of split pieces in their slots and the cross-CTA merge, then the final normalisation.  mutant
    restates one plausible kernel bug:
      "cacc not rescaled by corr", "zero-point term from unrounded P'", "merge weights from the other slot parity".
    Head 128 only.  Returns [rows, nH, head] in the model type."""
    assert case.head == HEAD
    mode, hpg, bias, E = case.mode, case.hpg, BIAS[case.mode], 2.0 ** P_EXP[case.mode]
    lens, meta = case.items()
    dec = A.decompose(lens, case.nG, grid, case.max_pieces)
    out = np.zeros((case.rows(), case.nH, case.head))
    slots = {}       # slot -> (item, g, M [nrow], L [nrow])
    partials = []    # (bg, [(slot_read, M, L, acc)] per piece, rows)
    for bg in dec.bgs:
        b, t0, nt = meta[bg.b]
        g = bg.g
        rows = [(b, t0 + r // hpg, g * hpg + r % hpg) for r in range(nt * hpg)]
        Lb = case.lens[b]
        S = np.stack([np.where(case.visible(b, tau), scores(case, data, b, g, data.q[b * case.q_len + tau, h][None])[0], -np.inf)
                      for b_, tau, h in rows])                                    # [nrow, Lb]
        sv = data.vs[b][:, g] * (E if mode != NONE else 1.0)
        bu = bias + data.vu[b][:, g] if mode in (I8, U4) else data.vc[b][:, g]   # what the P V MMA multiplies P' by
        bz = bias + data.vz[b][:, g]
        pieces = []
        for pc in bg.pieces:
            wm, wl, wo = [], [], []
            for w in range(4):
                m = np.full(len(rows), -np.inf); l = np.zeros(len(rows)); o = np.zeros((len(rows), case.head))
                cacc = np.zeros(len(rows))
                for t in range(pc.tok_lo, pc.tok_hi, 64):
                    lo, hi = t + 16 * w, min(t + 16 * w + 16, pc.tok_hi, Lb)
                    if lo >= hi:
                        continue
                    s = S[:, lo:hi]
                    mnew = np.maximum(m, s.max(1))
                    msub = np.where(mnew == -np.inf, 0.0, mnew)
                    corr = np.exp2(m - msub)
                    P = np.exp2(s - msub[:, None])
                    pq = rn32(P * rn32(sv[lo:hi])[None])
                    Pq = rn_f16(pq) if mode != NONE else (rn_ft(P, case.dtype) if case.dtype == BF16 else rn_f16(P))
                    l = l * corr + P.sum(1)
                    o = o * corr[:, None] + Pq @ bu[lo:hi]
                    if mode in (I8, U4):
                        cz = (pq if mutant == "zero-point term from unrounded P'" else Pq) @ bz[lo:hi]
                        cacc = (cacc if mutant == "cacc not rescaled by corr" else cacc * corr) + cz
                    m = mnew
                wm.append(m); wl.append(l * (E if mode != NONE else 1.0)); wo.append(o - cacc[:, None])
            M = np.max(wm, 0)
            f = [np.where(x == -np.inf, 0.0, np.exp2(x - np.where(M == -np.inf, 0.0, M))) for x in wm]
            L = sum(fi * li for fi, li in zip(f, wl))
            acc = sum(fi[:, None] * oi for fi, oi in zip(f, wo))
            if bg.npieces == 1:
                res = rn32(rn32(acc).astype(np.float32) / rn32(L)[:, None].astype(np.float32))
                for r, (b_, tau, h) in enumerate(rows):
                    out[b_ * case.q_len + tau, h] = res[r]
            else:
                slots[pc.slot_written] = (M, L)
                pieces.append((pc.slot_read, M, L, acc))
        if bg.npieces > 1:
            partials.append((bg, pieces, rows))
    for bg, pieces, rows in partials:
        Ms, Ls = [], []
        for slot, M, L, acc in pieces:
            if mutant == "merge weights from the other slot parity" and (slot ^ 1) in slots and len(slots[slot ^ 1][0]) == len(M):
                M, L = slots[slot ^ 1]
            Ms.append(M); Ls.append(L)
        Mg = np.max(Ms, 0)
        w = [np.where(x == -np.inf, 0.0, np.exp2(x - Mg)) for x in Ms]
        L = sum(wi * li for wi, li in zip(w, Ls))
        acc = sum(wi[:, None] * p[3] for wi, p in zip(w, pieces))
        res = rn32(rn32(acc).astype(np.float32) * (np.float32(1) / rn32(L)[:, None].astype(np.float32)))
        for r, (b_, tau, h) in enumerate(rows):
            out[b_ * case.q_len + tau, h] = res[r]
    return rn_ft(out, case.dtype)


# -------------------------------------------------------------------------------------------------- realistic data
def envelope(mode, dtype, q, kc, ks, vc, vs, kz, vis, alpha, depth, head=HEAD):
    """fp64 attention of one kv-group (q [rows, head] as the kernel reads it, K / V (c, s) [L, head] / [L], vis [rows, L])
    and the honest kernel's envelope with no absolute term:
      1/2 ulp_FT(ref) + u_P sum p|V| / l + (depth 2^-24 sum p s_v (BIAS + |c|) / l)  +  ln 2 |ds| sum p |V - ref| / l
    ds bounds the score error (fp32 score sums of `depth` steps, the fp16 conversion of Q in the quantized modes)."""
    bias = BIAS[mode]
    K = kc * ks[:, None]
    V = vc * vs[:, None]
    S = alpha * (q @ K.T)
    S = np.where(vis, S, -np.inf)
    E = np.exp(S - S.max(1, keepdims=True))
    l = E.sum(1, keepdims=True)
    ref = (E @ V) / l
    u_p = 2.0 ** -8 if (mode == NONE and dtype == BF16) else 2.0 ** -11
    accum = depth * 2.0 ** -24 * (E @ ((bias + np.abs(vc) + (256 if bias else 0)) * vs[:, None])) / l  # |u| <= |c| + |z|
    qa = np.abs(q)
    raw_mag = (qa @ ((bias + np.abs(kc) + np.abs(kz)[:, None]) * ks[:, None]).T)   # |sum q (BIAS + u)| + |(BIAS + z) sum q|
    ds = alpha * (raw_mag * (HEAD + 4) * 2.0 ** -24 + (2.0 ** -25 * HEAD * (bias + 448.0) * ks[None] if mode != NONE else 0.0))
    ds = ds + np.abs(S) * 2.0 ** -22
    Ed = E * np.where(vis, 2.0 * ds, 0.0)  # 2 ds: e^ds - 1 <= 2 ds for the ds in reach
    score = (Ed @ np.abs(V)) / l + np.abs(ref) * Ed.sum(1, keepdims=True) / l
    env = 0.5 * ulp_ft(ref, dtype) + u_p * (E @ np.abs(V)) / l + accum + score
    return ref, env


def tile_math(mode, q, kc, ks, vc, vs, vis, alpha, p_exp, dtype=BF16):
    """The quantized kernel's P V step restated (scores and sums in fp64): P = exp(s - max), P' = rn_f16(rn32(P s_v 2^E)),
    out = FT(sum P' c / (l 2^E)).  p_exp = 0 is the form before KVTraits::kPExp."""
    K = kc * ks[:, None]
    S = np.where(vis, alpha * (q @ K.T), -np.inf)
    P = np.exp(S - S.max(1, keepdims=True))
    Pq = rn_f16(rn32(P * rn32(vs * 2.0 ** p_exp)[None]))
    return rn_ft((Pq @ vc) / (P.sum(1, keepdims=True) * 2.0 ** p_exp), dtype)
