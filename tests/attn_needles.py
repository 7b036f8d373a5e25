"""Needle inputs for SpanAttention: single tokens that carry most of a head's softmax weight, so a token dropped, counted
twice or read one position off at a tile, span or split-KV piece edge moves the output far outside the tolerance.

With N(0,1) keys every token carries about 1/L of the weight, and at the long contexts where split-KV pieces and two-level
merges happen the attention tolerance cannot see one token.  Here R = 16 head dims are reserved:
  * ordinary tokens: K and V are N(0,1) outside the reserved dims and 0 inside them;
  * a needle for query head h at token j has the K row a' e_{d_h} (d_h: the head's reserved dim) with a' chosen so that
    its score is exactly ln L + C - drop (the row holds nothing else, so no N(0,1) term shifts it), and V[j, r] = MARK
    in a reserved dim r that no other needle of the head and neither neighbouring token marks, so each needle leaves its
    own mark in the output;
  * the query of head h is a * e_{d_h} plus N(0,1) outside the reserved dims, a = sqrt((ln L + C) * sqrt(head)), so the
    ordinary scores keep their usual spread and a needle with drop 0 scores exactly ln L + C.
Zeros survive every cache quantizer exactly (int8 / uint4: the code of 0 is the zero point; e4m3: code 0).

Also here, importable without the native library:
  * decompose(): a restatement of the work split at the top of span_attn_kernel (flat (sequence, kv-head, tile) list cut
    into ranges of Tc tiles, one per CTA; pieces, partial slots, direct and two-level merges);
  * evaluate(): fp64 attention over a dequantized cache with the per-element error envelope, the simulated rounding of an
    honest kernel and the "teeth" of every needle (how far removing or moving it moves the fp64 output).
"""
import math
from dataclasses import dataclass, field

import numpy as np
import torch

import kv_fp8_ref as F8
from oracle import kvcache_ref as KV

NONE, I8, U4, FP8 = KV.QUANT_NONE, KV.QUANT_I8, KV.QUANT_U4, F8.QUANT_FP8
MODE_NAMES = {NONE: "none", I8: "i8", U4: "u4", FP8: "fp8"}
TILE = 64             # tokens per tile of span_attn_kernel
MERGE_DIRECT = 16     # kMergeDirect: up to this many pieces the last CTA merges them all
MERGE_FAN = 8         # kMergeFan: above, groups of 8 pieces are merged first (level 1), then the groups
MERGE_MAX_SRC = 96    # kMergeMaxSrc: sources of one merge call
R = 16                # reserved head dims (one per query head of a kv-group: hpg <= 16)
C = 3.0               # needle score = ln L + C
MARK = 4.0            # value of a needle's V row in its marker dim
TEETH = 20.0          # a removed or moved needle must move its head's fp64 output by this many envelopes


# ------------------------------------------------------------------------------------------------ work decomposition
@dataclass
class Piece:
    cta: int
    tile_lo: int       # flat tile range [tile_lo, tile_hi) of the launch
    tile_hi: int
    tok_lo: int        # token range [tok_lo, tok_hi) of the sequence
    tok_hi: int
    slot_written: int  # partial slot the CTA stores to: 2 * cta + (piece does not start at the CTA's first tile)
    slot_read: int     # slot the merge reads: 2 * k0 + 2 * i (+ first_par for i == 0)


@dataclass
class Group:           # level-1 group of the two-level merge
    q: int
    first: int         # index of its first piece
    size: int
    lead: int          # slot of its first piece: level-1 counter and level-1 partial index


@dataclass
class BG:              # one (sequence, kv-head)
    b: int
    g: int
    start: int         # flat tile range [start, end)
    end: int
    k0: int
    npieces: int
    first_par: int
    pieces: list
    groups: list = field(default_factory=list)

    @property
    def merge(self):
        return "single" if self.npieces == 1 else ("direct" if self.npieces <= MERGE_DIRECT else "two-level")


@dataclass
class Decomposition:
    Tc: int
    total: int
    grid: int
    bgs: list

    def ctas(self):
        """cta -> [(bg, piece)] in the order the CTA processes them"""
        out = {}
        for bg in self.bgs:
            for pc in bg.pieces:
                out.setdefault(pc.cta, []).append((bg, pc))
        return out


def decompose(lens, n_groups, grid, max_pieces=None):
    """The split span_attn_kernel derives on the device from the lengths: total = n_groups * sum ceil(len_b / 64) tiles in
    b-major, then g, then tile order; Tc = max(ceil(total / grid), ceil(max_tiles / max_pieces), 1); CTA c covers tiles
    [c Tc, min(total, (c + 1) Tc)).  max_pieces: B2_ATTN_MAX_PIECES (None: unbounded)."""
    tiles = [(L + TILE - 1) // TILE for L in lens]
    total = n_groups * sum(tiles)
    mp = max_pieces if max_pieces else 1 << 20
    Tc = max(-(-total // grid), -(-max(tiles) // mp), 1)
    bgs, base = [], 0
    for b, tb in enumerate(tiles):
        for g in range(n_groups):
            s, e = base + g * tb, base + (g + 1) * tb
            k0 = s // Tc
            npieces = (e - 1) // Tc - k0 + 1
            first_par = 1 if s > k0 * Tc else 0
            pieces = []
            for i in range(npieces):
                cta = k0 + i
                lo, hi = max(s, cta * Tc), min(e, (cta + 1) * Tc)
                pieces.append(Piece(cta, lo, hi, (lo - s) * TILE, min(lens[b], (hi - s) * TILE),
                                    2 * cta + (1 if lo != cta * Tc else 0), 2 * k0 + 2 * i + (first_par if i == 0 else 0)))
            bg = BG(b, g, s, e, k0, npieces, first_par, pieces)
            if npieces > MERGE_DIRECT:
                for q in range(-(-npieces // MERGE_FAN)):
                    bg.groups.append(Group(q, q * MERGE_FAN, min(MERGE_FAN, npieces - q * MERGE_FAN),
                                           2 * (k0 + q * MERGE_FAN) + (first_par if q == 0 else 0)))
            bgs.append(bg)
        base += n_groups * tb
    return Decomposition(Tc, total, grid, bgs)


def check_decomposition(dec, lens):
    """The invariants the kernel's partial slots, counters and merges rely on (AssertionError if one fails)."""
    assert sum(bg.end - bg.start for bg in dec.bgs) == dec.total
    level0, leads = {}, {}
    for bg in dec.bgs:
        L = lens[bg.b]
        # the pieces tile the (sequence, kv-head) exactly, in tiles and in tokens
        assert bg.pieces[0].tile_lo == bg.start and bg.pieces[-1].tile_hi == bg.end, bg
        assert bg.pieces[0].tok_lo == 0 and bg.pieces[-1].tok_hi == L, bg
        for a, c in zip(bg.pieces, bg.pieces[1:]):
            assert a.tile_hi == c.tile_lo and a.tok_hi == c.tok_lo and c.cta == a.cta + 1, bg
        for i, pc in enumerate(bg.pieces):
            assert pc.tile_lo < pc.tile_hi and pc.tok_lo < pc.tok_hi and 0 <= pc.cta < dec.grid, (bg, pc)
            assert dec.Tc * pc.cta <= pc.tile_lo and pc.tile_hi <= dec.Tc * (pc.cta + 1), (bg, pc)
            if bg.npieces == 1:
                continue
            # only the first piece can start inside its CTA's range (slot parity 1); the merge reads what was written
            assert i == 0 or pc.slot_written % 2 == 0, (bg, pc)
            assert pc.slot_written == pc.slot_read, (bg, pc)
            assert pc.slot_written not in level0, ("level-0 slot written twice", bg, pc)
            level0[pc.slot_written] = bg
        assert bg.npieces <= dec.grid
        if bg.groups:
            assert len(bg.groups) <= MERGE_MAX_SRC
            assert sum(gr.size for gr in bg.groups) == bg.npieces and all(gr.size == MERGE_FAN for gr in bg.groups[:-1])
            for gr in bg.groups:
                assert gr.lead == bg.pieces[gr.first].slot_read, (bg, gr)
                assert gr.lead < 2 * dec.grid
                # level-1 counters and partials are indexed by the lead slot: no two groups of the launch may share one
                assert gr.lead not in leads, ("level-1 slot shared", bg, gr, leads[gr.lead])
                leads[gr.lead] = bg
    for cta, items in dec.ctas().items():
        slots = [pc.slot_written for bg, pc in items if bg.npieces > 1]
        assert len(slots) <= 2 and len(set(slots)) == len(slots), (cta, items)
        assert all(s // 2 == cta for s in slots)
        # a CTA's pieces other than its first and last are whole (sequence, kv-head)s: they need no partial slot
        for bg, pc in items[1:-1]:
            assert bg.npieces == 1, (cta, bg)


def shapes(dec):
    """Merge shapes present in a decomposition."""
    found = set()
    ctas = dec.ctas()
    for idx, bg in enumerate(dec.bgs):
        n = bg.npieces
        last_cta = bg.pieces[-1].cta
        next_shares = idx + 1 < len(dec.bgs) and dec.bgs[idx + 1].pieces[0].cta == last_cta
        if n == 1 and len(ctas[bg.pieces[0].cta]) > 2 and ctas[bg.pieces[0].cta][0][0] is not bg \
                and ctas[bg.pieces[0].cta][-1][0] is not bg:
            found.add("single inside a shared CTA")
        if n == 2 and bg.first_par:
            found.add("2 pieces, mid-CTA start")
        if n in (16, 17):
            found.add("%d pieces" % n)
        if n > MERGE_DIRECT and next_shares and n % MERGE_FAN in (0, 1):
            found.add("8q%s pieces, next starts in the last CTA" % ("" if n % MERGE_FAN == 0 else "+1"))
        if dec.Tc == 1 and n > 100:
            found.add("Tc = 1, > 100 pieces")
    return found


MERGE_SHAPES = {"single inside a shared CTA", "2 pieces, mid-CTA start", "16 pieces", "17 pieces",
                "8q pieces, next starts in the last CTA", "8q+1 pieces, next starts in the last CTA", "Tc = 1, > 100 pieces"}


def _len_of(tiles, rem):
    return TILE * (tiles - 1) + rem


def merge_shape_cases(grid):
    """(lens, nH, nG, max_pieces) of the merge-shape launches for a grid of `grid` CTAs (B2_ATTN_CTAS_PER_SM=1: the SM
    count).  Case 1 forces Tc = 4 through max_pieces and lays out, in flat tile order: 25 pieces ending inside a CTA that
    the next sequence starts in (8q+1: a last level-1 group of one piece), 24 pieces (8q) likewise, 2 pieces starting mid-CTA,
    a one-tile sequence inside a CTA shared by three, 17 pieces starting mid-CTA, 16 pieces.  Case 2 runs one sequence
    over nearly every CTA with Tc = 1."""
    tiles1 = [(98, 37), (92, 64), (3, 1), (1, 50), (63, 63), (60, 20)]
    case1 = ([_len_of(t, r) for t, r in tiles1], 8, 1, 25)
    case2 = ([_len_of(grid - 10, 59), 100], 16, 1, None)
    return [case1, case2]


# --------------------------------------------------------------------------------------------------- needle layout
def tile_and_span_edges(L, span):
    """0, L - 1 and the first and last token of every 64-token tile and of every span"""
    pos = {0, L - 1}
    for step in (TILE, span):
        for s in range(0, L, step):
            pos.add(s)
            pos.add(min(L, s + step) - 1)
    return sorted(pos)


def piece_edges(dec, bg):
    """first and last token of every piece, the last tile's first token, 0 and len - 1"""
    L = bg.pieces[-1].tok_hi
    pos = {0, L - 1, (L - 1) // TILE * TILE}
    for pc in bg.pieces:
        pos.add(pc.tok_lo)
        pos.add(pc.tok_hi - 1)
    return sorted(pos)


def schedule(positions, hpg, per_head):
    """Spread the needle positions of one (sequence, kv-head) over launches ("rounds"): each round gives each of the hpg
    query heads up to per_head needles, two needles of one head at least 2 tokens apart (so moving one by a token never
    lands on another).  Returns [[(head, pos), ...] per round]."""
    rounds, rest = [], list(positions)
    while rest:
        heads = [[] for _ in range(hpg)]
        left, h0 = [], 0
        for p in rest:
            for k in range(hpg):
                h = (h0 + k) % hpg
                if len(heads[h]) < per_head and (not heads[h] or p - heads[h][-1] >= 2):
                    heads[h].append(p)
                    h0 = h + 1
                    break
            else:
                left.append(p)
        rounds.append([(h, p) for h in range(hpg) for p in heads[h]])
        rest = left
    return rounds


def graded(dec, bg, hpg):
    """Needles of descending strength (drop 0, 1, 2) for query head 0 in the first piece, a middle level-1 group (or
    middle piece) and the last piece: their merge weights are O(1), so a wrong max correction or a dropped group shows."""
    pcs = bg.pieces
    if len(pcs) < 2:
        return []
    if bg.groups:
        mid = bg.groups[len(bg.groups) // 2]
        picks = [pcs[-1].tok_hi - 1, pcs[mid.first].tok_lo + 1, pcs[0].tok_lo]
    else:
        picks = [pcs[-1].tok_hi - 1, pcs[len(pcs) // 2].tok_lo + 1, pcs[0].tok_lo] if len(pcs) > 2 else [pcs[-1].tok_hi - 1, pcs[0].tok_lo]
    out, seen = [], set()
    for drop, p in enumerate(picks):
        if p not in seen and all(abs(p - s) >= 2 for s in seen):
            out.append((0, p, float(drop)))
            seen.add(p)
    return out


def amplitude(L, head):
    return math.sqrt((math.log(L) + C) * math.sqrt(head))


def to_type(x, dtype):
    """fp32 values of x rounded to the 16-bit model type (torch.bfloat16 / torch.float16)"""
    return torch.from_numpy(np.ascontiguousarray(x, np.float32)).to(dtype).float().numpy()


class Problem:
    """Seeded K / V rows and query noise of one launch.  rows(needles) places needles [(b, head, pos, drop)] and returns
    K and V rows per sequence [W_b, nG, head] and Q [B, nH, head], rounded to the model type.  written[b] >= lens[b] tokens are
    in the cache; attention reads lens[b]."""

    def __init__(self, lens, nH, nG, head, dtype, seed, written=None):
        self.lens, self.nH, self.nG, self.head, self.dtype = list(lens), nH, nG, head, dtype
        self.hpg = nH // nG
        assert self.hpg <= R
        self.written = list(written or lens)
        rng = np.random.default_rng(seed)
        self.kbase, self.vbase = [], []
        for W in self.written:
            k = rng.standard_normal((W, nG, head)).astype(np.float32)
            k[..., head - R:] = 0.0
            v = rng.standard_normal((W, nG, head)).astype(np.float32)
            v[..., head - R:] = 0.0
            self.kbase.append(to_type(k, dtype))
            self.vbase.append(to_type(v, dtype))
        self.qnoise = rng.standard_normal((len(lens), nH, head)).astype(np.float32)
        self.qnoise[..., head - R:] = 0.0

    def dim(self, h):
        return self.head - R + h % self.hpg

    def rows(self, needles):
        q = self.qnoise.copy()
        amp = [amplitude(L, self.head) for L in self.lens]
        for b in range(len(self.lens)):
            for h in range(self.nH):
                q[b, h, self.dim(h)] = amp[b]
        q = to_type(q, self.dtype)
        k = [x.copy() for x in self.kbase]
        v = [x.copy() for x in self.vbase]
        mark = {}  # (b, g, pos) -> marker dim, distinct from the marks of the head's other needles and of tokens pos +- 1
        for b, h, j, drop in sorted(needles, key=lambda n: n[2]):
            g = h // self.hpg
            score = math.log(self.lens[b]) + C - drop
            k[b][j, g] = 0.0
            k[b][j, g, self.dim(h)] = score * math.sqrt(self.head) / q[b, h, self.dim(h)]
            taken = {mark.get((b, g, j - 1)), mark.get((b, g, j + 1))}
            taken |= {mark[(b, g, p)] for bb, hh, p, _ in needles if (bb, hh) == (b, h) and (b, g, p) in mark}
            r = mark[(b, g, j)] = min(set(range(self.head - R, self.head)) - taken)
            v[b][j, g, r] = MARK
        return [to_type(x, self.dtype) for x in k], [to_type(x, self.dtype) for x in v], q


# ------------------------------------------------------------------------------------------------------------ caches
def quantize(x, mode):
    """The CPU cache quantizers: x fp32 [..., 128] -> (c, s) with the cached value c * s in fp64.  c is what the kernel's
    P V MMA multiplies: the value itself (bf16 / fp16 cache), q - zero (int8 / uint4), e4m3(code) (fp8); s is the scale."""
    x = np.asarray(x, np.float32)
    if mode == NONE:
        return x.astype(np.float64), np.ones(x.shape[:-1])
    if mode in (I8, U4):
        q, z, s = KV.quant_rows(x, mode)
        return q.astype(np.float64) - z[..., None].astype(np.float64), s.astype(np.float64)
    codes, _, s = F8.quant_rows(x)
    return F8.decode(codes).astype(np.float64), s.astype(np.float64)


def from_spans(spans, mode, span, nG, W, head, dtype):
    """(c, s) as above, [nG, W, head] and [nG, W], read from span bytes (a list of uint8 arrays, one per span)."""
    c = np.zeros((nG, W, head))
    s = np.ones((nG, W))
    for si in range((W + span - 1) // span):
        buf, n = spans[si], min(span, W - si * span)
        sl = slice(si * span, si * span + n)
        if mode == NONE:
            v = buf[:nG * span * head * 2].view(np.uint16).reshape(nG, span, head)[:, :n]
            c[:, sl] = KV.bits_to_f32(v) if dtype == torch.bfloat16 else v.view(np.float16).astype(np.float32)
            continue
        row = head // 2 if mode == U4 else head
        d = buf[:nG * span * row].reshape(nG, span, row)[:, :n]
        prm = buf[nG * span * row:nG * span * (row + 8)].view(np.float32).reshape(nG, span, 2)[:, :n]
        if mode == I8:
            q = d.view(np.int8).astype(np.float64)
        elif mode == U4:
            q = np.stack([d & 0xF, d >> 4], -1).reshape(nG, n, head).astype(np.float64)
        else:
            q = F8.decode(d).astype(np.float64)
        c[:, sl] = q - prm[..., 0:1].astype(np.float64)
        s[:, sl] = prm[..., 1]
    return c, s


# ------------------------------------------------------------------------------------------------- oracle + envelope
def p_type(mode, dtype, head):
    """(unit roundoff of the probabilities the P V MMA multiplies, absolute error floor of their subnormals).
    head 128: bf16 cache -> P in bf16 (exponent range of fp32: no subnormals in reach); fp16 cache -> P in fp16; int8 /
    uint4 / fp8 -> P * s_v in fp16 (tile_compute_q folds the V scale into P).  fp16 subnormals are spaced 2^-24, so a
    rounded value is off by at most 2^-25 absolutely.  head 64: P stays fp32."""
    if head != 128:
        return 2.0 ** -24, 0.0
    if mode == NONE and dtype == torch.bfloat16:
        return 2.0 ** -8, 0.0
    return 2.0 ** -11, 2.0 ** -25


def _round_p(x, mode, dtype, head):
    x = x.astype(np.float32)
    if head != 128:
        return x.astype(np.float64)
    if mode == NONE and dtype == torch.bfloat16:
        return to_type(x, torch.bfloat16).astype(np.float64)
    return x.astype(np.float16).astype(np.float64)


@dataclass
class Result:
    ref: np.ndarray        # [B, nH, head] fp64 attention
    env: np.ndarray        # [B, nH, head] per-element bound
    honest: float          # max |simulated honest kernel - ref| / env
    teeth: float           # min over needles of max_d |mutated ref - ref| / env
    weakest: tuple         # the needle (and mutation) with the least teeth


def evaluate(prob, q, kc, ks, vc, vs, mode, needles, alpha=None, stale=()):
    """fp64 attention over the dequantized cache (kc * ks, vc * vs per sequence, [nG, W, head]) of the first lens[b]
    tokens, with
      env = 2e-3 + rel |ref| + u_P sum_t p_t |V_t| + f_P sum_t |c_t| / l
    rel: the existing contract (bf16 2^-7, fp16 2^-9, covering the output rounding); u_P, f_P: p_type; l: the softmax
    denominator relative to the global max.  `honest` repeats the kernel's rounding: P (or P * s_v) rounded to the P type
    from the fp32 value, the output rounded once to the model type.  `teeth` is the least, over the needles, of the
    output change when the needle is removed or moved to token j - 1 / j + 1 (its K row swapped with the neighbour's),
    and, for `stale` needles [(b, h, pos)] beyond lens[b], when token pos is attended too."""
    head, hpg = prob.head, prob.hpg
    alpha = alpha if alpha is not None else 1.0 / math.sqrt(head)
    rel = 2.0 ** -9 if prob.dtype == torch.float16 else 2.0 ** -7
    u_p, f_p = p_type(mode, prob.dtype, head)
    B = len(prob.lens)
    ref = np.zeros((B, prob.nH, head))
    env = np.zeros_like(ref)
    honest, teeth, weakest = 0.0, math.inf, None
    by_head = {}
    for b, h, j, _ in needles:
        by_head.setdefault((b, h), []).append(j)
    stale_by_head = {}
    for b, h, j in stale:
        stale_by_head.setdefault((b, h), []).append(j)
    qd = q.astype(np.float64)
    for b in range(B):
        L = prob.lens[b]
        for g in range(prob.nG):
            K = kc[b][g] * ks[b][g][:, None]
            V = vc[b][g, :L] * vs[b][g, :L, None]
            hs = list(range(g * hpg, (g + 1) * hpg))
            S = alpha * (K @ qd[b, hs].T)                   # [W, hpg]
            M = S[:L].max(0)
            E = np.exp(S - M)                               # rows >= L: stale tokens (not attended)
            e = E[:L]
            l = e.sum(0)
            o = (e.T @ V) / l[:, None]
            ev = 2e-3 + rel * np.abs(o) + u_p * (e.T @ np.abs(V)) / l[:, None] + f_p * np.abs(vc[b][g, :L]).sum(0)[None] / l[:, None]
            ref[b, hs], env[b, hs] = o, ev
            P = _round_p(e * vs[b][g, :L, None], mode, prob.dtype, head)
            sim = to_type((P.T @ vc[b][g, :L]) / l[:, None], prob.dtype)
            honest = max(honest, float((np.abs(sim - o) / ev).max()))
            for i, h in enumerate(hs):
                for j in by_head.get((b, h), []):
                    if L < 2 or j >= L:  # a stale needle's teeth: below
                        continue
                    muts = [("removed", (o[i] * l[i] - e[j, i] * V[j]) / (l[i] - e[j, i]))]
                    for k in (j - 1, j + 1):
                        if 0 <= k < L:
                            muts.append(("moved to %d" % k, o[i] + (e[k, i] - e[j, i]) * (V[j] - V[k]) / l[i]))
                    for what, mo in muts:
                        r = float((np.abs(mo - o[i]) / ev[i]).max())
                        if r < teeth:
                            teeth, weakest = r, (b, h, j, what)
                for x in stale_by_head.get((b, h), []):
                    vx = vc[b][g, x] * vs[b][g, x]
                    mo = (o[i] * l[i] + E[x, i] * vx) / (l[i] + E[x, i])
                    r = float((np.abs(mo - o[i]) / ev[i]).max())
                    if r < teeth:
                        teeth, weakest = r, (b, h, x, "stale token attended")
    return Result(ref, env, honest, teeth, weakest)


def cpu_caches(k_rows, v_rows, mode):
    """(kc, ks, vc, vs) per sequence, [nG, W, head] / [nG, W], of the CPU quantizers' cache of these rows"""
    out = ([], [], [], [])
    for b in range(len(k_rows)):
        kc, ks = quantize(k_rows[b], mode)
        vc, vs = quantize(v_rows[b], mode)
        for lst, x in zip(out, (kc.transpose(1, 0, 2), ks.T, vc.transpose(1, 0, 2), vs.T)):
            lst.append(x)
    return out


# --------------------------------------------------------------------------------------------------------- the cases
@dataclass
class Case:
    name: str
    mode: int
    dtype: object
    span: int
    nH: int
    nG: int
    lens: list
    head: int = 128
    per_head: int = 4            # needles per query head and launch
    written: list = None         # tokens written per sequence (stale rows beyond lens)
    fill: int = 0                # byte the span pool starts with
    max_pieces: int = None       # B2_ATTN_MAX_PIECES
    ctas_per_sm: int = None      # B2_ATTN_CTAS_PER_SM
    layout: str = "tiles"        # needle positions: "tiles", "pieces", "stale", "head64"
    seed: int = 0

    @property
    def hpg(self):
        return self.nH // self.nG

    def problem(self):
        return Problem(self.lens, self.nH, self.nG, self.head, self.dtype, self.seed, self.written)

    def rounds(self, grid):
        """[(needles [(b, h, pos, drop)], stale [(b, h, pos)])] per launch.  grid: CTAs of the attention handle."""
        B, hpg = len(self.lens), self.hpg
        if self.layout == "stale":
            return [self._stale_round()]
        dec = decompose(self.lens, self.nG, grid, self.max_pieces) if self.head == 128 else None
        per_bg = {}
        for b, L in enumerate(self.lens):
            for g in range(self.nG):
                if self.layout == "tiles":
                    pos = tile_and_span_edges(L, self.span)
                elif self.layout == "head64":
                    pos = sorted({0, L - 1, min(31, L - 1), min(32, L - 1)} | set(tile_and_span_edges(L, self.span)))
                else:
                    pos = piece_edges(dec, dec.bgs[b * self.nG + g])
                per_bg[(b, g)] = schedule(pos, hpg, self.per_head)
        n = max(len(r) for r in per_bg.values())
        out = []
        for r in range(n):
            nd = []
            for (b, g), rr in per_bg.items():
                if r < len(rr):
                    nd += [(b, g * hpg + h, p, 0.0) for h, p in rr[r]]
            out.append((nd, []))
        if self.layout == "pieces":
            nd = []
            for bg in dec.bgs:
                nd += [(bg.b, bg.g * hpg + h, p, drop) for h, p, drop in graded(dec, bg, hpg)]
            if nd:
                out.append((nd, []))
        return out

    def _stale_round(self):
        """heads 0 / 1 of every group: needles only at stale tokens (token lens[b], and a later span); the other heads:
        needles at the tile and span edges of [0, lens[b])"""
        nd, st = [], []
        for b, L in enumerate(self.lens):
            W = self.written[b]
            later = min(W - 1, (L // self.span + 2) * self.span + 5)
            for g in range(self.nG):
                h0 = g * self.hpg
                nd += [(b, h0, L, 0.0), (b, h0 + 1, later, 0.0)]
                st += [(b, h0, L), (b, h0 + 1, later)]
                live = schedule(tile_and_span_edges(L, self.span), self.hpg - 2, self.per_head)
                assert len(live) == 1, "one launch must hold every live needle"
                nd += [(b, h0 + 2 + h, p, 0.0) for h, p in live[0]]
        return nd, st


BF16, FP16 = torch.bfloat16, torch.float16
TILE_LENS = [1, 63, 64, 65, 777, 2049, 4100]


def tile_cases():
    """Needles on every tile and span edge, default knobs: each length alone and all of them as one ragged batch, in
    every cache mode and both model types, spans 16 / 128, heads 28/4 and 16/1."""
    out = []
    for mode in (NONE, I8, U4, FP8):
        for dtype in (BF16, FP16):
            for span in (16, 128):
                for nH, nG in ((28, 4), (16, 1)):
                    for lens in [[L] for L in TILE_LENS] + [TILE_LENS[::-1]]:
                        name = "%s-%s-s%d-%d/%d-%s" % (MODE_NAMES[mode], "fp16" if dtype == FP16 else "bf16", span, nH, nG,
                                                      "ragged" if len(lens) > 1 else lens[0])
                        out.append(Case(name, mode, dtype, span, nH, nG, lens, seed=len(out)))
    return out


def merge_cases(grid, mode=NONE, dtype=BF16):
    """The merge shapes at B2_ATTN_CTAS_PER_SM=1 (grid = the SM count): needles on the first and last token of every
    piece, then one launch of graded needles"""
    out = []
    for i, (lens, nH, nG, mp) in enumerate(merge_shape_cases(grid)):
        out.append(Case("merge%d-%s" % (i + 1, MODE_NAMES[mode]), mode, dtype, 16, nH, nG, lens, max_pieces=mp, ctas_per_sm=1,
                        layout="pieces", seed=100 + i))
    return out


def long_cases():
    """ctx 32768 (the maximum of config C2), alone and next to a 5000-token sequence: needles at 0, len - 1, the last tile
    and every piece edge of the default grid"""
    out = []
    for mode in (NONE, I8, FP8):
        for lens in ([32768], [32768, 5000]):
            out.append(Case("ctx32768-%s-B%d" % (MODE_NAMES[mode], len(lens)), mode, BF16, 128, 28, 4, lens, layout="pieces",
                            seed=200 + mode * 2 + len(lens)))
    return out


def stale_cases():
    """L2 = 300 tokens written, attention over L1 = 100 (mid-tile) and 128 (a tile start)"""
    return [Case("stale-%s" % MODE_NAMES[mode], mode, BF16, 16, 28, 4, [100, 128], written=[300, 300], layout="stale",
                 seed=300 + mode) for mode in (NONE, I8, U4, FP8)]


def head64_cases():
    """head 64, bf16 spans, 0xFF-filled pool: hpg 1, 7 (the warps loop twice) and 16"""
    return [Case("head64-%d/%d" % (nH, nG), NONE, BF16, 16, nH, nG, [1, 31, 32, 33, 1000], head=64, per_head=8, fill=0xFF,
                 layout="head64", seed=400 + nH) for nH, nG in ((2, 2), (14, 2), (16, 1))]
