"""CPU restatement of b2_penalize and of the token history (include/b200spark.h), in numpy.

The processor is restated from the contract over the plain [B, max_len] history (the reference's in_ids / cur_len /
input_len), not over the kernel's per-id table, so a wrong table update shows up as a wrong logit.  Values are carried in
fp64 and rounded to FT with round-to-nearest-even (torch's conversion); every FT operation of the contract is exact in
fp64 before its one rounding, except the quotient of the repetition penalty.  The kernel's quotient comes from
div.approx.f32 (bf16) or rcp.approx.ftz.f32 (fp16), within about 2^-22 relative of the exact one, so where the exact
quotient lies within DIV_REL of an FT rounding boundary both neighbours are accepted (`penalize` returns them as `alt`).

`bugs` restates one wrong processor each (BUGS); the CPU suite shows that every one of them changes an output."""
import numpy as np
import torch

FTS = {"bf16": torch.bfloat16, "fp16": torch.float16}
DIV_REL = 2.0 ** -20
BAN = -1e9
IN_PROMPT = 1 << 30

BUGS = ["rep_not_rounded", "zero_multiplies", "duplicate_twice", "prompt_counted", "suppress_ignored", "freq_first",
        "ngram_off_by_one", "min_len_generated", "fp16_ban_finite", "outside_shard"]


def rn(v, ft):
    """fp64 values -> the nearest FT values (ties to even), as fp64"""
    return torch.as_tensor(np.asarray(v, np.float64)).to(FTS[ft]).double().numpy()


def bits(v, ft):
    """FT values (fp64 holding FT values) -> uint16 bits"""
    return torch.as_tensor(np.asarray(v, np.float64)).to(FTS[ft]).view(torch.int16).numpy().view(np.uint16)


def values(b, ft):
    """uint16 bits -> fp64 values"""
    return torch.from_numpy(np.asarray(b, np.uint16).view(np.int16).copy()).view(FTS[ft]).double().numpy()


def f32(v):
    return np.float32(v)


def ftz(v):
    """an fp32 value with a subnormal flushed to a zero of its sign (the reference's .ftz arithmetic)"""
    v = np.float32(v)
    return np.float32(np.copysign(0.0, v)) if v != 0 and abs(v) < np.float32(2.0 ** -126) else v


def penalty_sum(cnt, freq, pres):
    """s = fl32(cnt freq) (+ presence when cnt > 0), fp32 with subnormals flushed"""
    with np.errstate(all="ignore"):
        s = ftz(f32(ftz(f32(cnt)) * ftz(f32(freq))))
        if cnt > 0:
            s = ftz(f32(s + ftz(f32(pres))))
    return s


def _div(x, r, ft):
    """(RN(x / r), the other acceptable result): exact quotient in fp64, ambiguous within DIV_REL of a boundary"""
    with np.errstate(all="ignore"):
        q = np.float64(x) / np.float64(r)
    y = rn(q, ft)
    if np.isfinite(q) and q != 0:
        lo, hi = rn(q * (1 - DIV_REL), ft), rn(q * (1 + DIV_REL), ft)
        return y, (lo if lo != y else hi)
    return y, y


def penalize(x, tokens, lens, prompt_lens, params, ft, id_offset=0, bugs=()):
    """x: fp64 [rows, n] FT values of vocabulary ids [id_offset, id_offset + n); tokens [rows, >= L] ints.  params: dict of
    per-row lists repetition, presence, frequency, no_repeat_ngram, min_length, eos_id, suppress.  Returns (out, alt): the
    processed values and, where the quotient is ambiguous, the other acceptable value (alt == out elsewhere)."""
    bugs = set(bugs)
    out = np.array(x, np.float64, copy=True)
    alt = out.copy()
    rows, n = out.shape
    ban = np.float64(-65504.0) if ft == "fp16" and "fp16_ban_finite" in bugs else rn(BAN, ft)[()]

    def col(t):
        c = int(t) - id_offset
        if "outside_shard" in bugs:
            return c % n
        return c if 0 <= c < n else None

    for r in range(rows):
        L, P = int(lens[r]), int(prompt_lens[r])
        hist = [int(t) for t in tokens[r][:L]]
        R = rn(params["repetition"][r], ft)[()] if "rep_not_rounded" not in bugs else np.float64(np.float32(params["repetition"][r]))
        sup = int(params["suppress"][r]) != 0 and "suppress_ignored" not in bugs
        freq, pres = params["frequency"][r], params["presence"][r]
        gen_from = 0 if "prompt_counted" in bugs else P
        occurring = {}
        for j, t in enumerate(hist):
            if 0 <= t:
                occurring.setdefault(t, 0)
                if j >= gen_from:
                    occurring[t] += 1
        cnt_gen = {}
        for j in range(P, L):
            cnt_gen[hist[j]] = cnt_gen.get(hist[j], 0) + 1
        visits = []
        for t in occurring:
            visits += [t] * (2 if "duplicate_twice" in bugs and len([u for u in hist if u == t]) > 1 else 1)
        for t in visits:
            c = col(t)
            if c is None:
                continue
            v, va = out[r, c], alt[r, c]
            cnt = occurring[t]

            def rep_step(v):
                if R == 1 or (sup and cnt_gen.get(t, 0) == 0):
                    return v, v
                neg = v <= 0 if "zero_multiplies" in bugs else v < 0
                if neg:
                    with np.errstate(all="ignore"):
                        y = rn(v * R, ft)[()]
                    return y, y
                if "rep_not_rounded" in bugs:
                    with np.errstate(all="ignore"):
                        y = rn(np.float64(np.float32(np.float32(v) / np.float32(R))), ft)[()]
                    return y, y
                return _div(v, R, ft)

            def pen_step(v):
                pen = rn(penalty_sum(cnt, freq, pres), ft)[()]
                if pen == 0 and not np.signbit(pen):
                    return v
                with np.errstate(all="ignore"):
                    return rn(v - pen, ft)[()]

            if "freq_first" in bugs:
                v1 = pen_step(v)
                v, va = rep_step(v1)
            else:
                v1, v1a = rep_step(v)
                v, va = pen_step(v1), pen_step(v1a)
            out[r, c], alt[r, c] = v, va
        g = int(params["no_repeat_ngram"][r])
        bans = []
        if g > 0:
            last = L - g - (1 if "ngram_off_by_one" in bugs else 0)
            for j in range(0, last + 1):
                if hist[j:j + g - 1] == hist[L - g + 1:L]:
                    bans.append(hist[j + g - 1])
        eos = int(params["eos_id"][r])
        cur = L - P if "min_len_generated" in bugs else L
        if cur < int(params["min_length"][r]) and eos >= 0:
            bans.append(eos)
        for t in bans:
            c = col(t) if t >= 0 else None
            if c is not None:
                out[r, c] = alt[r, c] = ban
    return out, alt


def same(a, b):
    """element-wise: equal FT bits, or both NaN"""
    return (a == b) & ~(np.isnan(a) | np.isnan(b)) & (np.signbit(a) == np.signbit(b)) | (np.isnan(a) & np.isnan(b))


def rows_and_params(rows, n, rng):
    """per-row histories and parameters: empty, prompt-only, generation-only, heavy duplicates, ids 0 and n - 1, EOS in and
    out of the history, n-grams of 0 .. 4 with matches at the first and last admissible j, min_length at L - 1, L, L + 1,
    penalties -2 / 0 / 2 and repetition 0.5 / 1 / 1.05 / 2"""
    hists, prompts = [], []
    prm = {k: [] for k in neutral(0)}
    reps, pens = [0.5, 1.0, 1.05, 2.0, 0.0], [-2.0, 0.0, 2.0, 0.5]
    for r in range(rows):
        kind = r % 6
        L = [0, 40, 40, 60, 3, 200][kind]
        if kind == 3:    # heavy duplicates
            h = rng.integers(0, min(n, 4), L)
        else:
            h = rng.integers(0, n, L)
        if kind == 4 or kind == 5:
            h[:2] = [0, n - 1][:len(h[:2])]
        if kind == 5 and n > 20:  # the NaN, +inf and -inf columns of make_logits
            h[2:5] = [7, 9, 10]
        g = r % 5
        if g >= 2 and L >= 2 * g:  # plant the last g - 1 tokens at j = 0 and at j = L - g (the first and last admissible j)
            tail = h[L - g + 1:]
            h[:g - 1] = tail
            h[L - g:L - 1] = tail
        P_len = {0: 0, 1: L, 2: 0}.get(kind, L // 2)
        hists.append(h)
        prompts.append(P_len)
        prm["repetition"].append(reps[r % len(reps)])
        prm["presence"].append(pens[r % 4])
        prm["frequency"].append(pens[(r // 4) % 4])
        prm["no_repeat_ngram"].append(g)
        prm["min_length"].append(L + (r % 3) - 1)
        prm["eos_id"].append(int(h[-1]) if (r % 2 and L) else (n - 1 if r % 4 == 0 else -1))
        prm["suppress"].append(r % 3 == 1)
    return hists, prompts, prm


def make_logits(rows, n, ft, rng):
    x = rng.standard_normal((rows, n)) * 3
    x[:, ::11] = 0.0
    x[:, 1::13] = -0.0
    if n > 20:
        x[::2, 7] = np.nan
        x[1::3, 9] = np.inf
        x[2::3, 10] = -np.inf
    return rn(x, ft)


def case(ft, n, rows):
    """the inputs of one (ft, n, rows) case of the GPU comparison, from a fixed seed: (histories, prompt lengths, params,
    logits as fp64 FT values)"""
    rng = np.random.default_rng(n * 131 + rows)
    hists, prompts, prm = rows_and_params(rows, n, rng)
    return hists, prompts, prm, make_logits(rows, n, ft, rng)


CASES = [(ft, n, rows) for rows in (1, 64, 65) for n in (1, 7, 4097, 152064) for ft in ("bf16", "fp16")]


class History:
    """The token history's bookkeeping (load / append / reset), restated per slot from its definition."""

    def __init__(self, rows, max_len, vocab):
        self.rows, self.max_len, self.vocab = rows, max_len, vocab
        self.tokens = [[] for _ in range(rows)]
        self.prompt = [0] * rows

    def load(self, slot, ids, prompt_len=None):
        ids = [int(t) for t in ids]
        assert len(ids) <= self.max_len
        self.tokens[slot] = [t if 0 <= t < self.vocab else -1 for t in ids]
        self.prompt[slot] = len(ids) if prompt_len is None else prompt_len

    def reset(self, slot):
        self.load(slot, [], 0)

    def append(self, ids):
        for r, t in enumerate(ids):
            if len(self.tokens[r]) < self.max_len:
                self.tokens[r].append(int(t) if 0 <= t < self.vocab else -1)

    def table(self, slot):
        """{id: entry} for the ids of the slot (bit 30: in the prompt, low bits: generated count)"""
        e = {}
        for j, t in enumerate(self.tokens[slot]):
            if t < 0:
                continue
            e[t] = e.get(t, 0) | (IN_PROMPT if j < self.prompt[slot] else 0)
            e[t] += j >= self.prompt[slot]
        return e

    def arrays(self):
        """(tokens [rows, max_len] with -1 padding, lens, prompt_lens) for `penalize`"""
        tok = np.full((self.rows, self.max_len), -1, np.int64)
        for r, t in enumerate(self.tokens):
            tok[r, :len(t)] = t
        return tok, np.array([len(t) for t in self.tokens]), np.array(self.prompt)


def neutral(rows):
    return dict(repetition=[1.0] * rows, presence=[0.0] * rows, frequency=[0.0] * rows, no_repeat_ngram=[0] * rows,
                min_length=[0] * rows, eos_id=[-1] * rows, suppress=[0] * rows)
