"""Exact-arithmetic inputs and a restatement of the weight-only GEMM kernels (wq_gemm.cu, wq_gemv2.cu, wq_gemm_tc.cu), so a
test can hold every output element to ONE rounding instead of the 2e-2 of the random-data tests.

Importable without the native library or a GPU.

Inputs.  Activations are a = j * 2^-e with integer |j| <= J; zero points are z = i * 2^-pz; scales are s = m * 2^-(ps + r)
with m in 1..7 and r in 0..2; dense bf16 weights are i * 2^-f.  The kernels multiply the activations with integer codes c
(W4: b0 + q; W8: 17 b0 + u, u = q (+128 for int8: the sign flip of the image); b0 = 16 for bf16 handles, 128 for fp16,
`prepare_impl` in wq_gemm.cu) and apply the affine dequantization to the fp32 accumulator.  precondition() checks, on the
actual data, that every partial sum the kernels can form (any order, any split-K or cluster slice, the fixed-order reducer)
is a multiple of its grid unit and stays below 2^23 units: then the fp32 accumulation is exact whatever the tensor cores
do, even if they align addends with one bit less than fp32.  It also checks that every named intermediate of the epilogue
(z' * sum a, acc - z' sum a, s * (...), alpha * v, + bias, + residual) is an fp32 number, so those operations are exact
in either FMA-contracted or separate form.  The last rounding is then the single FT store.

What this excludes: fp16 W8 handles (c up to 17 * 143 = 2431) at K above about 3400 with J = 1, and K * J * 31 >= 2^23
for bf16 W4 (K > 67000 at J = 4).  The generator refuses such inputs (ValueError) instead of producing inexact ones.

Restatement after accumulation (read off the kernels):
  * per-channel, every kernel (split-K GEMV, gemv2, wgmma):  v = s * (acc - z' * sum a),  z' = z + zbias (pack_sz_kernel);
  * sub-channel on the mma.sync GEMV:  v = sum_g s_g * (acc_g - z'_g * sum_g a)  (wq_gemm_kernel, GROUPED fold);
  * sub-channel on wgmma (GROUPED, group_tiles and the per-word group_k look-up): every weight rounded to FT once,
    w = rn(fma(q - 8, s, rn(rn32((8 - z) s)))), then an exact accumulation;
  * epilogue: alpha, + bias, activation, + residual, one FT rounding; SwiGLU: silu(g alpha) * (u alpha).
With the exact inputs all of this is exact up to the activation (__expf, tanhf, erff: act_bound()) and the
final FT rounding.  expected() returns the fp64 value y before the rounding and a bound E on the fp32 error before it; an
honest kernel stores a value in [rn(y - E), rn(y + E)] (E = 0: exactly rn(y)).

Also here: a copy of the host dispatch (launches()), so every test case states which kernel it reaches.
"""
from dataclasses import dataclass, field

import numpy as np

KBK, KBN = 64, 128          # k per tile, channels per tile (wq_gemm_shared.cuh)
GEMV_MAX_M = 16             # kGemvMaxM
TC_MAX_M = 64               # kTcMaxM: rows per wgmma launch
TC_MIN_M = 17               # kTcMinM
TC_MAX_SPLIT = 6            # B2_GEMM_TC_MAX_SPLIT default
H100_SMS = 132
LIMIT = 2.0 ** 23           # partial sums stay below this many grid units
ACT_NONE, ACT_TANH, ACT_GELU_ERF, ACT_GELU_TANH, ACT_RELU, ACT_SILU, ACT_SIGMOID = 0, 1, 2, 3, 4, 5, 6
ACT_SWIGLU = 7
EXACT_ACTS = (ACT_NONE, ACT_RELU)


@dataclass
class Case:
    """One GEMM handle: weight width, FT ('bf16' / 'fp16'), group size (-1: per channel), shape, int8 signedness, pair."""
    wbits: int
    K: int
    N: int
    group: int = -1
    ft: str = "bf16"
    signed: bool = True
    pair: bool = False

    @property
    def b0(self):
        return 128 if self.ft == "fp16" else 16

    @property
    def grouped(self):
        return self.wbits != 16 and self.group != -1

    @property
    def group_k(self):    # general group size (not a multiple of 64): the wgmma kernel at every batch
        return self.group if self.grouped and self.group % KBK else 0

    @property
    def KT(self):
        kq = self.group if (self.grouped and not self.group_k) else KBK
        return (self.K + kq - 1) // kq * kq // KBK

    @property
    def NG(self):
        return (self.N + 63) // 64 if self.pair else (self.N + KBN - 1) // KBN

    @property
    def G(self):
        return (self.K + self.group - 1) // self.group if self.grouped else 1

    def name(self):
        g = "pc" if self.group == -1 else f"g{self.group}"
        return f"w{self.wbits}-{g}-{self.ft}-K{self.K}-N{self.N}" + ("-pair" if self.pair else "") + ("" if self.signed else "-u8")


# --------------------------------------------------------------------------------------------------- FT rounding
def rn_ft(x, ft):
    """Round fp64 values to the FT (round to nearest even), returned as fp64.  The values must be fp32 numbers (every caller
    passes exact ones), so the fp32 step in between is not a second rounding."""
    import torch
    x = np.asarray(x, np.float64)
    x32 = x.astype(np.float32)
    assert np.array_equal(x32.astype(np.float64), x), "rn_ft needs fp32-exact inputs"
    dt = torch.float16 if ft == "fp16" else torch.bfloat16
    return torch.from_numpy(x32).to(dt).to(torch.float64).numpy()


def ulp_ft(y, ft):
    """Unit in the last place of |y| in the FT (fp16 subnormals included)."""
    a = np.abs(np.asarray(y, np.float64))
    ex = np.floor(np.log2(np.where(a > 0, a, 1.0)))
    if ft == "fp16":
        return np.exp2(np.maximum(ex, -14) - 10)
    return np.exp2(np.maximum(ex, -126) - 7)


def bound_units(y, E, ft):
    """The per-element bound of an assertion: half an FT ulp of the result plus the fp32 error E before the rounding."""
    return 0.5 * ulp_ft(np.abs(y) + E, ft) + E


def is_f32(x):
    x = np.asarray(x, np.float64)
    return np.array_equal(x.astype(np.float32).astype(np.float64), x)


# --------------------------------------------------------------------------------------------------- inputs
@dataclass
class Weights:
    q: np.ndarray            # [K, N] int64 logical codes (int8 signed, uint8 / uint4 unsigned); dense: None
    s: np.ndarray = None     # [G, N] fp64 (FT values)
    z: np.ndarray = None     # [G, N] fp64 (FT values)
    w: np.ndarray = None     # dense [K, N] fp64 (FT values)
    unit_s: float = 1.0
    unit_z: float = 1.0
    unit_w: float = 1.0      # dense weights' grid


def make_weights(case, seed, pz=None, ps=None, f=10):
    r = np.random.default_rng(seed)
    K, N = case.K, case.N
    if case.wbits == 16:
        w = r.integers(-96, 97, size=(K, N)).astype(np.float64) * 2.0 ** -f
        return Weights(q=None, w=w, unit_w=2.0 ** -f)
    G = case.G
    if case.wbits == 4:
        q = r.integers(0, 16, size=(K, N))
        pz = 1 if pz is None else pz
        z = r.integers(0, 15 * 2 ** pz + 1, size=(G, N)) * 2.0 ** -pz
        ps = 8 if ps is None else ps
    else:
        q = r.integers(-128, 128, size=(K, N)) if case.signed else r.integers(0, 256, size=(K, N))
        pz = 0 if pz is None else pz
        lo, hi = (-8, 8) if case.signed else (120, 136)
        z = r.integers(lo * 2 ** pz, hi * 2 ** pz + 1, size=(G, N)) * 2.0 ** -pz
        ps = 11 if ps is None else ps
    s = r.integers(1, 8, size=(G, N)) * np.exp2(-(ps + r.integers(0, 3, size=(G, N))))
    return Weights(q=q.astype(np.int64), s=s, z=z, unit_s=2.0 ** -(ps + 2), unit_z=2.0 ** -pz)


def make_acts(M, K, J=3, e=3, seed=0):
    r = np.random.default_rng(seed)
    return r.integers(-J, J + 1, size=(M, K)).astype(np.float64) * 2.0 ** -e


def onehot_acts(ks, K, value=1.0):
    """Row m is value * e_{ks[m]}: out[m, n] reads back the dequantized weight (ks[m], n)."""
    A = np.zeros((len(ks), K))
    A[np.arange(len(ks)), np.asarray(ks)] = value
    return A


def make_vec(n, seed, scale=2.0 ** -6, J=64):
    r = np.random.default_rng(seed)
    return r.integers(-J, J + 1, size=n).astype(np.float64) * scale


def pack_qdata(case, wt):
    """The C ABI's weight layout: int4 [K, ceil(N/2)] (low nibble = even column), int8 / uint8 [K, N], bf16 / fp16 [K, N]."""
    if case.wbits == 4:
        q = wt.q.astype(np.uint8)
        if case.N % 2:
            q = np.concatenate([q, np.zeros((case.K, 1), np.uint8)], axis=1)
        return ((q[:, 1::2] << 4) | (q[:, 0::2] & 0xF)).astype(np.uint8)
    if case.wbits == 8:
        return wt.q.astype(np.int8 if case.signed else np.uint8)
    return wt.w


# --------------------------------------------------------------------------------------------------- restatement
def group_index(case, K=None):
    """Quantization group of every k (general groups: one look-up per 8-k word, which never straddles a group)."""
    k = np.arange(case.K if K is None else K)
    if not case.grouped:
        return np.zeros_like(k)
    return np.minimum(k // case.group, case.G - 1)


def dequant_exact(case, wt, gidx=None):
    """(q - z) s per weight, fp64 exact; dense weights as they are."""
    if case.wbits == 16:
        return wt.w.copy()
    g = group_index(case) if gidx is None else gidx
    return (wt.q - wt.z[g]) * wt.s[g]


def dequant_tc_grouped(case, wt, gidx=None, zero=None):
    """Weights as the wgmma GROUPED dequantization produces them: (b0 + q) - (b0 + 8) = q - 8 exactly, then
    fma.rn(q - 8, s, rn_FT(rn32((b0 + 8 - (z + b0)) s))): one FT rounding per weight."""
    g = group_index(case) if gidx is None else gidx
    z = wt.z if zero is None else zero
    zz = (case.b0 + 8.0 - (z + case.b0))                           # fp32: exact for dyadic zero points
    c32 = (zz * wt.s).astype(np.float32).astype(np.float64)        # fp32 product (exact: few bits)
    gc = rn_ft(c32, case.ft)
    x = (wt.q - 8.0) * wt.s[g] + gc[g]
    return rn_ft(x, case.ft)


def path_weights(case, wt, path):
    """The fp64 weight matrix whose exact product with A a path computes (before its epilogue)."""
    return dequant_tc_grouped(case, wt) if (path == "tc" and case.grouped) else dequant_exact(case, wt)


def _act(x, act):
    f32 = lambda c: float(np.float32(c))
    if act in (ACT_NONE,):
        return x
    if act == ACT_RELU:
        return np.maximum(x, 0.0)
    if act == ACT_TANH:
        return np.tanh(x)
    if act == ACT_GELU_ERF:
        from scipy.special import erf
        return x * 0.5 * (1.0 + erf(x * f32(0.70710678)))
    if act == ACT_GELU_TANH:
        return x * 0.5 * (1.0 + np.tanh(f32(0.7978845608028654) * (x + f32(0.044715) * x * x * x)))
    if act == ACT_SILU:
        return x / (1.0 + np.exp(-x))
    if act == ACT_SIGMOID:
        return 1.0 / (1.0 + np.exp(-x))
    raise ValueError(act)


U24 = 2.0 ** -24             # half an fp32 ulp, relative


def act_bound(x, y, act):
    """fp32 error of the kernels' activation forms (b2_common.cuh apply_act) at fp32 input x, result y, from the CUDA math
    library's maximum errors: __expf 2 + floor(1.173 |x|) ulp, tanhf and erff 2 ulp; every other operation one rounding."""
    ax, ay = np.abs(x), np.abs(y)
    if act in EXACT_ACTS:
        return np.zeros_like(ay)
    if act in (ACT_SILU, ACT_SIGMOID):      # x / (1 + __expf(-x)), 1 / (1 + __expf(-x)): relative to y; below
        E = (2 * (3 + 1.2 * ax) + 4) * U24 * ay  # x = -88.72 (-x log2 e >= 128) __expf(-x) is inf and the result zero
        return np.where(x < -88.72, np.maximum(E, ay), E)
    if act == ACT_TANH:                     # tanhf
        return 6 * U24 * ay
    if act == ACT_GELU_ERF:                 # x * 0.5 * (1 + erff(x * c)): erff's absolute error and the rounding of x * c
        return 0.5 * ax * (8 * U24 + 1.2 * ax * U24) + 4 * U24 * ay
    if act == ACT_GELU_TANH:                # x * 0.5 * (1 + tanhf(c1 (x + c2 x^3))): five roundings inside the argument
        arg = 0.8 * (ax + 0.045 * ax ** 3)
        return 0.5 * ax * (8 * U24 + 6 * U24 * arg) + 4 * U24 * ay
    raise ValueError(act)


def expected(A, W, act=ACT_NONE, alpha=1.0, bias=None, res=None, W2=None, res_first=False):
    """fp64 result before the FT store and its fp32 error bound E (0 where the epilogue is exact).  W2: the up weights of a
    SwiGLU pair (W the gate).  res_first: the residual added before the activation (a mutation, not a kernel)."""
    x = alpha * (A @ W)
    if W2 is not None:
        return swiglu(x, alpha * (A @ W2))
    if bias is not None:
        x = x + bias[None, :]
    if res is not None and res_first:
        x = x + res
    y = _act(x, act)
    E = act_bound(x, y, act)
    if res is not None and not res_first:
        y = y + res
    return y, E


def swiglu(g, u):
    """silu(g) * u of the pair epilogue (g, u already scaled by alpha) and its bound: silu's, times |u|, plus the product."""
    sg = _act(g, ACT_SILU)
    y = sg * u
    return y, act_bound(g, sg, ACT_SILU) * np.abs(u) + 2 * U24 * np.abs(y)


def check(out, y, E, ft):
    """out (fp64 of the stored FT values) against y / E: returns (bad mask, deviation in bound units)."""
    out = np.asarray(out, np.float64)
    exact = E == 0
    lo = np.where(exact, y, y - E - 2.0 ** -22 * np.abs(y))
    hi = np.where(exact, y, y + E + 2.0 ** -22 * np.abs(y))
    lo_r = rn_ft(lo.astype(np.float32).astype(np.float64), ft)
    hi_r = rn_ft(hi.astype(np.float32).astype(np.float64), ft)
    bad = ~((out >= lo_r) & (out <= hi_r)) | np.isnan(out)
    dev = np.abs(out - y) / bound_units(y, E, ft)
    return bad, dev


def teeth(y, E, y_mut, ft):
    """How far a mutated restatement lands from the honest one, in units of the honest bound (max over elements)."""
    return float(np.max(np.abs(y_mut - y) / bound_units(y, E, ft)))


# --------------------------------------------------------------------------------------------------- exactness precondition
def precondition(case, wt, A, path, alpha=1.0, bias=None, res=None, act=ACT_NONE, unit_a=None, unit_b=2.0 ** -6, W2wt=None):
    """Raise ValueError unless every fp32 intermediate of `path` is exact for these inputs (see the module docstring).
    Returns the largest partial-sum magnitude in units of LIMIT (< 1)."""
    absA = np.abs(A)
    if unit_a is None:
        nz = absA[absA > 0]
        unit_a = float(np.exp2(np.floor(np.log2(nz.min())))) if nz.size else 1.0
        while not np.all(np.mod(A / unit_a, 1.0) == 0):
            unit_a /= 2
    worst = 0.0
    for w in ([wt] if W2wt is None else [wt, W2wt]):
        if case.wbits == 16:
            if not np.all(np.mod(w.w / w.unit_w, 1.0) == 0):
                raise ValueError("dense weights off their grid")
            worst = max(worst, (absA @ np.abs(w.w)).max() / (unit_a * w.unit_w) / LIMIT)
            v = A @ w.w
        elif path == "tc" and case.grouped:
            W = dequant_tc_grouped(case, w)
            nzw = np.abs(W[W != 0])
            unit_w = 1.0
            if nzw.size:
                unit_w = float(np.exp2(np.floor(np.log2(nzw.min()))))
                while not np.all(np.mod(W / unit_w, 1.0) == 0):
                    unit_w /= 2
            worst = max(worst, (absA @ np.abs(W)).max() / (unit_a * unit_w) / LIMIT)
            v = A @ W
        else:
            g = group_index(case)
            cmax = case.b0 + 15 if case.wbits == 4 else 17 * (case.b0 + 15)
            codes_bound = absA.sum(1).max() * cmax / unit_a / LIMIT          # sum a c, every partial, both W8 planes
            zb = case.b0 if case.wbits == 4 else (17 * case.b0 + (128 if case.signed else 0))
            zp = w.z + zb                                                     # z' (fp32 exact: z dyadic)
            sa_bound = absA.sum(1).max() / unit_a / LIMIT
            zsa = 0.0
            vb = 0.0
            for gi in range(case.G):
                ks = g == gi
                sa = A[:, ks].sum(1)                                          # [M]
                prod = sa[:, None] * zp[gi][None, :]
                if not is_f32(prod):
                    raise ValueError("z' * sum a is not an fp32 number")
                zsa = max(zsa, (np.abs(sa)[:, None] * np.abs(zp[gi])[None, :]).max() / (unit_a * w.unit_z) / LIMIT)
                d = A[:, ks] @ (w.q[ks] - w.z[gi][None, :] * 1.0)
                if not is_f32(d) or not is_f32(d * w.s[gi][None, :]):
                    raise ValueError("acc - z' sum a or its scaled value is not an fp32 number")
                vb = max(vb, (absA[:, ks] @ np.abs(w.q[ks] - w.z[gi][None, :]) * w.s[gi][None, :]).max()
                         / (unit_a * w.unit_z * w.unit_s) / LIMIT)
            worst = max(worst, codes_bound, sa_bound, zsa, vb)
            v = A @ dequant_exact(case, w)
        if worst >= 1.0:
            raise ValueError(f"partial sums reach {worst:.3f} x 2^23 grid units: not exact in fp32")
        x = alpha * v
        if not (is_f32(v) and is_f32(x)):
            raise ValueError("alpha * v is not an fp32 number")
        if bias is not None:
            x = x + bias[None, :]
            if not is_f32(x):
                raise ValueError("+ bias is not exact in fp32")
        if res is not None and act in EXACT_ACTS:
            if not is_f32(_act(x, act) + res):
                raise ValueError("+ residual is not exact in fp32")
    return worst


# --------------------------------------------------------------------------------------------------- fp8 activations
# b2_gemm_wq_run_fp8 (wq_gemm_tc_kernel<4, MULTI, true>): the activations are quantized per row by b2_quant_fp8
# (scale = amax / 448 in fp32, codes = rn_e4m3(x * fp32(1 / scale)), tile_sums = per-64-k sums of the codes); the int4 codes q
# become exact e4m3 numbers (nib4_to_e4m3) and the e4m3 MMAs run into a separate accumulator dt that is added to the fp32 d
# every 128 k (two weight tiles).  The Hopper e4m3 MMA keeps fewer than fp32's bits while it accumulates, so the exact-input
# precondition here is stronger: within every two consecutive 64-k tiles sum |y q| < 2^12 units (or a single nonzero
# product), i.e. the inputs rely on no more than 13 bits of the fp8 accumulation.  After the accumulation the kernel computes
#   part = fp32(fp32(s * scale_m) * (d - z * sum_tiles y))      (A8: zz = z' - 16 = z)
# per k-slice, sums the S partials in slice order in fp32, and runs the epilogue; all of it is restated in fp32 here.
FP8_WINDOW = 2.0 ** 12


def quant_fp8(x):
    """b2_quant_fp8 restated bit for bit: codes y (fp64 of the e4m3 values), scale [M] fp32, tile_sums [M, KT] fp32."""
    import torch
    xf = np.asarray(x, np.float64).astype(np.float32)
    sc = (np.maximum(np.abs(xf).max(axis=1), np.float32(1e-12)) / np.float32(448)).astype(np.float32)
    rs = (np.float32(1) / sc).astype(np.float32)
    y = torch.from_numpy((xf * rs[:, None]).astype(np.float32)).to(torch.float8_e4m3fn).double().numpy()
    K = xf.shape[1]
    ts = np.stack([y[:, k:k + KBK].sum(1) for k in range(0, K, KBK)], 1).astype(np.float32)
    return y, sc, ts


def fp8_acts(M, K, J=2, seed=0, kstar=5):
    """x = j / 8 (|j| <= J) and x[:, kstar] = 56: every row's scale is 56 / 448 = 1/8 exactly, its codes are j and 448."""
    A = make_acts(M, K, J, 3, seed)
    A[:, kstar] = 56.0
    return A


def fp8_weights(case, seed, kstar=5):
    """int4 per-channel weights with q[kstar] = 0: the code 448 of the activations' amax column meets weight code 0, so the
    e4m3 MMAs only see the small codes (the zero-point term still carries it, in fp32)."""
    wt = make_weights(case, seed)
    wt.q[kstar] = 0
    return wt


def fp8_partials(case, wt, y, sc, S, q=None, ts_shift=0):
    """fp32 k-slice partials of the A8 kernel, summed in slice order.  q / ts_shift: mutations (other codes; the zero-point
    term read from the tile sums ts_shift tiles further on)."""
    q = wt.q if q is None else q
    f = lambda a: np.asarray(a, np.float64).astype(np.float32)
    ss = f(wt.s[0][None, :] * f(sc)[:, None].astype(np.float64))            # fp32(s * scale_m)
    K = case.K
    ts = np.stack([y[:, k:k + KBK].sum(1) for k in range(0, K, KBK)], 1)
    acc = np.zeros((y.shape[0], case.N), np.float32)
    for kt0, kt1 in tc_slices(case, S):
        k0, k1 = kt0 * KBK, min(kt1 * KBK, K)
        d = y[:, k0:k1] @ q[k0:k1].astype(np.float64)
        nt = ts.shape[1]
        sa = ts[:, [min(t + ts_shift, nt - 1) for t in range(kt0, kt1)]].sum(1)
        diff = d - wt.z[0][None, :] * sa[:, None]
        if not is_f32(d) or not is_f32(diff):
            raise ValueError("fp8 accumulator not exact in fp32")
        part = (ss * f(diff)).astype(np.float32)
        acc = part if S == 1 else (acc + part).astype(np.float32)
    return acc


def restate_fp8(case, wt, x, S, act=ACT_NONE, alpha=1.0, bias=None, res=None, wt2=None, **mut):
    """y, E of b2_gemm_wq_run_fp8 on activations x (fp64 of bf16 values).  E = 0: y is the fp32 value the kernel rounds."""
    assert alpha in (1.0, 0.5), "alpha * partial must stay exact"
    y8, sc, _ = quant_fp8(x)
    fs = fp8_partials(case, wt, y8, sc, S, **mut)
    if wt2 is not None:
        return swiglu(fs.astype(np.float64) * alpha, fp8_partials(case, wt2, y8, sc, S, **mut).astype(np.float64) * alpha)
    v = (fs * np.float32(alpha)).astype(np.float32)
    if bias is not None:
        v = (v + bias[None, :].astype(np.float32)).astype(np.float32)
    v64 = v.astype(np.float64)
    if act in EXACT_ACTS:
        out = _act(v64, act).astype(np.float32)
        if res is not None:
            out = (out + res.astype(np.float32)).astype(np.float32)
        return out.astype(np.float64), np.zeros(out.shape)
    y = _act(v64, act)
    E = act_bound(v64, y, act)
    return (y + res if res is not None else y), E


def precondition_fp8(case, wt, x, wt2=None):
    """Raise ValueError unless the e4m3 accumulation of every 128-k window and the fp32 sums are exact (see above)."""
    y, sc, ts = quant_fp8(x)
    K = case.K
    for w in [wt] + ([wt2] if wt2 is not None else []):
        ab = np.abs(y)
        worst = 0.0
        for k0 in range(0, K, KBK):
            win = slice(k0, min(k0 + 2 * KBK, K))
            prod = ab[:, win] @ w.q[win].astype(np.float64)
            single = ((ab[:, win] > 0)[:, :, None] & (w.q[win] > 0)[None]).sum(1) <= 1
            worst = max(worst, float(np.where(single, 0.0, prod).max()) / FP8_WINDOW)
        if worst >= 1.0:
            raise ValueError(f"an e4m3 128-k window reaches {worst:.2f} x 2^12 units")
        if (ab @ w.q.astype(np.float64)).max() >= LIMIT or (ab.sum(1) * np.abs(w.z).max()).max() >= LIMIT:
            raise ValueError("fp8 partial sums not exact in fp32")
    return worst


# --------------------------------------------------------------------------------------------------- host dispatch copy
def use_tc(case, M):
    """use_tc (wq_gemm.cu): general group sizes at every batch; else M >= 17 unless sub-channel int8."""
    if case.group_k:
        return True
    return M >= TC_MIN_M and (not case.grouped or case.wbits == 4)


def mt_index_for(M):
    return 0 if M <= 8 else 1


def tc_split(case, sms=H100_SMS, max_split=TC_MAX_SPLIT, ctas_per_sm=1):
    """make_tc_plan: S = slots / NG, at most KT / 4 and max_split, at least 1."""
    S = ctas_per_sm * sms // case.NG
    S = min(S, case.KT // 4, max_split)
    return max(S, 1)


def tc_slices(case, S):
    """k-tile ranges of the S k-slices of a wgmma unit: [s KT / S, (s + 1) KT / S)."""
    return [(s * case.KT // S, (s + 1) * case.KT // S) for s in range(S)]


def gemv2_cb(case, M, sms=H100_SMS, forced=0):
    """gemv2_plan's channel block (None: the split-K kernel runs instead)."""
    if M > GEMV_MAX_M:
        return None
    rows = case.NG * KBN
    cb_min = 32 if case.pair else 16
    cb = forced or 128
    if not forced:
        while cb > cb_min and rows // cb < 2 * sms:
            cb >>= 1
    if cb < cb_min or cb > 128 or (cb & (cb - 1)):
        return None
    if not forced and rows // cb < sms // 2:
        return None
    return cb


def launches(case, M, env=None, sms=H100_SMS, a8=False, norm_self=False):
    """The kernel launches of one b2_gemm_wq_run call (run_impl / run_tc): a list of dicts with the kernel's name as the
    profiler shows it, its rows and the facts that select a code path (wgmma: nm, MULTI, tc_S).  norm_self: the
    self-contained RMSNorm form, which only the split-K GEMV implements (dense bf16 included)."""
    env = env or {}
    H = "true" if case.ft == "fp16" else "false"
    out = []
    if a8:                                  # b2_gemm_wq_run_fp8: the e4m3 wgmma kernel at every batch
        S = tc_split(case, sms, int(env.get("B2_GEMM_TC_MAX_SPLIT", TC_MAX_SPLIT)))
        multi = case.NG * S > sms
        for m0 in range(0, M, TC_MAX_M):
            rows = min(TC_MAX_M, M - m0)
            out.append(dict(path="tc8", kernel=f"wq_gemm_tc_kernel<4, {'true' if multi else 'false'}, true, false, false>",
                            m0=m0, rows=rows, nm=32 if rows <= 32 else 64, multi=multi, S=S))
        return out
    if use_tc(case, M):
        S = tc_split(case, sms, int(env.get("B2_GEMM_TC_MAX_SPLIT", TC_MAX_SPLIT)))
        multi = case.NG * S > sms
        G = "true" if case.grouped else "false"
        for m0 in range(0, M, TC_MAX_M):
            rows = min(TC_MAX_M, M - m0)
            out.append(dict(path="tc", kernel=f"wq_gemm_tc_kernel<{case.wbits}, {'true' if multi else 'false'}, false, {G}, {H}>",
                            m0=m0, rows=rows, nm=32 if rows <= 32 else 64, multi=multi, S=S))
        return out
    if case.wbits == 16 and case.ft == "bf16" and M <= GEMV_MAX_M and not norm_self and env.get("B2_GEMV2", "1") != "0":
        cb = gemv2_cb(case, M, sms, int(env.get("B2_GEMV2_CB", 0)))
        if cb is not None:
            return [dict(path="gemv2", kernel=f"wq_gemv2_kernel<{1 if M <= 8 else 2}>", m0=0, rows=M, cb=cb)]
    split = ("forced" if int(env.get("B2_GEMM_FORCE_SPLIT", 0)) > 0 else
             "global" if env.get("B2_GEMM_CLUSTER", "1") == "0" else "planned")
    G = "true" if case.grouped else "false"
    for m0 in range(0, M, GEMV_MAX_M):
        rows = min(GEMV_MAX_M, M - m0)
        mt = 1 << mt_index_for(rows)
        out.append(dict(path="gemv", kernel=f"wq_gemm_kernel<{case.wbits}, {mt}, {G}, {H}>", m0=m0, rows=rows, mt=mt, split=split))
    return out


# --------------------------------------------------------------------------------------------------- read-back k sets
def sampled_ks(case, seed=0):
    """k values that reach every k-tile, chunk, word and nibble position of the image, every group start (and the word
    before it) and the whole K tail, for shapes too large to sweep every k."""
    r = np.random.default_rng(seed)
    K = case.K
    ks = set(range(min(KBK, K)))                       # one whole tile: every chunk / word / nibble / byte
    ks.update(range(max(0, K - KBK), K))               # the tail tile
    for kt in range((K + KBK - 1) // KBK):             # one k per 8-k word position, random nibble, in every tile
        w = kt * 8 + (kt % 8)
        if w * 8 < K:
            ks.add(min(K - 1, w * 8 + int(r.integers(0, 8))))
    if case.grouped:
        for g0 in range(0, K, case.group):
            ks.update(k for k in (g0 - 1, g0, g0 + 7, g0 + 8) if 0 <= k < K)
    return sorted(ks)


# --------------------------------------------------------------------------------------------------- GPU case list
@dataclass
class GpuCase:
    """One dyadic GEMM of the GPU suite.  path: the kernel it must reach ('gemv', 'gemv2', 'tc'); env: knobs set before
    the handle is created."""
    id: str
    case: Case
    M: int
    path: str
    env: dict = field(default_factory=dict)
    act: int = ACT_NONE
    alpha: float = 1.0
    bias: bool = False
    res: bool = False
    J: int = 3
    e: int = 3

    @property
    def a8(self):
        return self.path == "tc8"


def _gc(id_, case, M, path, **kw):
    return GpuCase(id_, case, M, path, **kw)


QWEN7B = [(3584, 4608), (3584, 3584), (3584, 18944), (18944, 3584)]
Q72_TP8 = [(8192, 1280), (1024, 8192), (3696, 8192)]

DYADIC_CASES = [
    # split-K GEMV: MT 1 and 2, W 4/8/16, per channel and g64/g128/g256, bf16 and fp16
    _gc("gemv-w4-pc-m1", Case(4, 3584, 4608), 1, "gemv", bias=True),
    _gc("gemv-w4-pc-m8-act", Case(4, 3584, 3584), 8, "gemv", act=ACT_GELU_TANH, alpha=-0.75, bias=True, res=True),
    _gc("gemv-w4-pc-m16-fp16", Case(4, 1024, 1023, ft="fp16"), 16, "gemv", bias=True, res=True),
    _gc("gemv-w8-pc-m3", Case(8, 3584, 3584), 3, "gemv", alpha=0.5, res=True, J=1),
    _gc("gemv-w8-pc-m12-fp16", Case(8, 1024, 640, ft="fp16"), 12, "gemv", J=1),
    _gc("gemv-w8-u8-m4", Case(8, 1024, 520, signed=False), 4, "gemv", act=ACT_TANH, J=1),
    _gc("gemv-w16-m5", Case(16, 1024, 520), 5, "gemv", env={"B2_GEMV2": "0"}, act=ACT_SIGMOID, bias=True),
    _gc("gemv-w4-g64-m9", Case(4, 1088, 777, group=64), 9, "gemv", act=ACT_RELU, res=True),
    _gc("gemv-w4-g128-m16", Case(4, 4096, 1024, group=128), 16, "gemv", alpha=-0.75, bias=True),
    _gc("gemv-w8-g256-m2-fp16", Case(8, 1024, 384, group=256, ft="fp16"), 2, "gemv", J=1),
    _gc("gemv-w8-g128-m7", Case(8, 2048, 640, group=128), 7, "gemv", act=ACT_GELU_ERF, J=1),
    # split forms of the GEMV: global split with workspace + ticket, forced split, clusters (default)
    _gc("gemv-w4-forced7", Case(4, 1024, 256), 2, "gemv", env={"B2_GEMM_FORCE_SPLIT": "7"}, bias=True, res=True),
    _gc("gemv-w4-g128-noclus", Case(4, 2048, 5118, group=128), 9, "gemv", env={"B2_GEMM_CLUSTER": "0"}, act=ACT_SILU, res=True, alpha=0.5),
    _gc("gemv-w4-cluster", Case(4, 2048, 5117), 7, "gemv", act=ACT_TANH, bias=True, res=True, alpha=0.5),
    _gc("gemv-w16-cluster", Case(16, 2048, 5117), 3, "gemv", env={"B2_GEMV2": "0"}, act=ACT_TANH, bias=True, res=True, alpha=0.5),
    _gc("gemv-w8-cluster", Case(8, 2048, 5117), 16, "gemv", act=ACT_TANH, bias=True, res=True, alpha=0.5, J=1),
    # sub-channel int8 above M = 16: 16-row passes on the mma.sync kernel
    _gc("gemv-w8-g128-m17", Case(8, 1024, 640, group=128), 17, "gemv", J=1, res=True),
    _gc("gemv-w8-g64-m33", Case(8, 1024, 384, group=64), 33, "gemv", J=1, act=ACT_RELU, bias=True),
    _gc("gemv-w8-g128-m40", Case(8, 2048, 520, group=128), 40, "gemv", J=1),
    # gemv2 (dense bf16, no split-K), every channel block
    *[_gc(f"gemv2-cb{cb}", Case(16, 1032, 640), m, "gemv2", env={"B2_GEMV2_CB": str(cb)}, bias=True, res=True,
          act=ACT_SILU if cb == 64 else ACT_NONE) for cb, m in ((16, 1), (32, 8), (64, 11), (128, 16))],
    # wgmma: N32 / N64, single unit and MULTI, tc_S, tail launches, epilogues
    _gc("tc-w4-m17", Case(4, 3584, 4608), 17, "tc", bias=True),
    _gc("tc-w4-m32-act", Case(4, 3584, 3584), 32, "tc", act=ACT_GELU_ERF, alpha=-0.75, res=True),
    _gc("tc-w4-m33", Case(4, 18944, 3584), 33, "tc", res=True, J=1),
    _gc("tc-w4-m64-multi", Case(4, 3584, 18944), 64, "tc", act=ACT_SIGMOID),
    _gc("tc-w8-m64", Case(8, 3584, 4608), 64, "tc", bias=True, res=True, J=1),
    _gc("tc-w8-m20-fp16", Case(8, 1024, 1023, ft="fp16"), 20, "tc", bias=True, J=1, act=ACT_TANH),
    _gc("tc-w16-m40", Case(16, 1024, 4100), 40, "tc", bias=True, act=ACT_SILU),
    _gc("tc-w4-q72-qkv", Case(4, 8192, 1280), 64, "tc", bias=True, J=2),
    _gc("tc-w4-q72-o", Case(4, 1024, 8192), 17, "tc", res=True, act=ACT_RELU),
    _gc("tc-w4-q72-down", Case(4, 3696, 8192), 48, "tc", res=True, alpha=0.5),
    _gc("tc-w4-tail65", Case(4, 1024, 1290), 65, "tc", res=True, bias=True),
    _gc("tc-w4-tail72", Case(4, 1024, 1290), 72, "tc", act=ACT_GELU_TANH),
    _gc("tc-w4-tail80-fp16", Case(4, 1024, 1290, ft="fp16"), 80, "tc", res=True),
    _gc("tc-w8-tail96", Case(8, 1024, 1290), 96, "tc", alpha=-0.75, J=1),
    _gc("tc-w4-m128", Case(4, 1024, 1290), 128, "tc", bias=True, res=True),
    _gc("tc-w4-split1", Case(4, 3584, 4608), 40, "tc", env={"B2_GEMM_TC_MAX_SPLIT": "1"}, bias=True),
    # sub-channel on wgmma: group_tiles (g128, g256) and per-word general groups (g40, g72, g200) incl. M = 1
    _gc("tc-g128-m32", Case(4, 4096, 1024, group=128), 32, "tc", res=True, J=2),
    _gc("tc-g256-m64-fp16", Case(4, 2048, 1023, group=256, ft="fp16"), 64, "tc", bias=True, J=2),
    _gc("tc-g40-m1", Case(4, 1000, 1023, group=40), 1, "tc", act=ACT_SILU, J=2),
    _gc("tc-g72-m17", Case(4, 2048, 1023, group=72), 17, "tc", res=True, J=2),
    _gc("tc-g200-m40-fp16", Case(4, 1000, 1023, group=200, ft="fp16"), 40, "tc", bias=True, res=True, J=2),
    _gc("tc-g40-m70", Case(4, 1000, 520, group=40), 70, "tc", alpha=0.5, J=2),
    # SwiGLU pairs on the GEMV, gemv2 and wgmma (N not a multiple of 64)
    _gc("pair-gemv-w4", Case(4, 1024, 704, pair=True), 5, "gemv"),
    _gc("pair-gemv-w4-g128", Case(4, 1024, 704, group=128, pair=True), 16, "gemv", J=2),
    _gc("pair-gemv2", Case(16, 1024, 704, pair=True), 3, "gemv2", env={"B2_GEMV2_CB": "32"}),
    _gc("pair-tc-w4", Case(4, 3584, 18944, pair=True), 64, "tc", J=2),
    _gc("pair-tc-w8", Case(8, 1024, 1000, pair=True), 33, "tc", J=1),
    _gc("pair-tc-g128", Case(4, 1024, 1000, group=128, pair=True), 20, "tc", J=2),
]

# Weight read-back: small shapes sweep every k; large ones the sampled set
READBACK_CASES = [
    _gc("rb-gemv-w4-pc", Case(4, 520, 130), 16, "gemv"),
    _gc("rb-gemv-w4-pc-m8-fp16", Case(4, 520, 130, ft="fp16"), 8, "gemv"),
    _gc("rb-gemv-w8-pc", Case(8, 328, 77), 16, "gemv"),
    _gc("rb-gemv-w8-u8", Case(8, 328, 77, signed=False), 8, "gemv"),
    _gc("rb-gemv-w4-g64", Case(4, 200, 130, group=64), 16, "gemv"),
    _gc("rb-gemv-w8-g128", Case(8, 520, 130, group=128), 16, "gemv"),
    _gc("rb-gemv-w16", Case(16, 520, 130), 16, "gemv", env={"B2_GEMV2": "0"}),
    _gc("rb-gemv2", Case(16, 520, 640), 16, "gemv2", env={"B2_GEMV2_CB": "16"}),
    _gc("rb-tc-w4-pc", Case(4, 520, 130), 64, "tc"),
    _gc("rb-tc-w4-pc-n32", Case(4, 520, 130), 32, "tc"),
    _gc("rb-tc-w8-pc", Case(8, 520, 130), 64, "tc"),
    _gc("rb-tc-w8-pc-fp16", Case(8, 520, 130, ft="fp16"), 33, "tc"),
    _gc("rb-tc-w16", Case(16, 520, 130), 40, "tc"),
    _gc("rb-tc-g128", Case(4, 520, 130, group=128), 64, "tc"),
    _gc("rb-tc-g40", Case(4, 520, 130, group=40), 64, "tc"),
    _gc("rb-tc-g72-fp16", Case(4, 520, 130, group=72, ft="fp16"), 64, "tc"),
    _gc("rb-tc-g200-m1", Case(4, 1000, 130, group=200), 1, "tc"),
    _gc("rb-pair-gemv", Case(4, 520, 130, pair=True), 16, "gemv"),
    _gc("rb-pair-tc", Case(4, 520, 130, pair=True), 64, "tc"),
    _gc("rb-pair-gemv2", Case(16, 520, 130, pair=True), 16, "gemv2", env={"B2_GEMV2_CB": "32"}),
    # large shapes: the sampled k set
    _gc("rbs-tc-w4-qwen-qkv", Case(4, 3584, 4608), 64, "tc"),
    _gc("rbs-gemv-w4-qwen-down", Case(4, 18944, 3584), 16, "gemv"),
    _gc("rbs-tc-w8-qwen-o", Case(8, 3584, 3584), 64, "tc"),
    _gc("rbs-tc-g128-q72-down", Case(4, 3696, 8192, group=128), 64, "tc"),
    _gc("rbs-gemv-w8-g128", Case(8, 4096, 1280, group=128), 16, "gemv"),
]


def call_form(i):
    """Call form of dyadic case i: (lda - K, ldc - N, element offset of the C view).  Strided views, an odd ldc and a C view
    that is not 4-byte aligned (the generic epilogues), in turn; ldc > N always, so every row has guard columns."""
    return [(0, 4, 0), (8, 8, 0), (64, 1, 0), (8, 4, 1), (64, 8, 0)][i % 5]


def readback_ks(gc):
    return list(range(gc.case.K)) if gc.case.K <= 1100 else sampled_ks(gc.case, seed=len(gc.id))


def _seed(gc):
    return sum(map(ord, gc.id))


def dyadic_inputs(gc):
    """The inputs of one GPU case (the same on every machine): weights (two sets for a pair), A, bias, residual."""
    sd = _seed(gc)
    c = gc.case
    mk = fp8_weights if gc.a8 else make_weights
    wt = mk(c, sd)
    wt2 = mk(c, sd + 1) if c.pair else None
    A = fp8_acts(gc.M, c.K, gc.J, sd + 2) if gc.a8 else make_acts(gc.M, c.K, gc.J, gc.e, sd + 2)
    bias = make_vec(c.N, sd + 3) if gc.bias else None
    res = make_vec(gc.M * c.N, sd + 4).reshape(gc.M, c.N) if gc.res else None
    return dict(wt=wt, wt2=wt2, A=A, bias=bias, res=res)


def restate(gc, inp, W=None, W2=None, sms=H100_SMS, **mut):
    """y, E of a GPU case from its inputs (W / W2: the path weights, computed if not given; fp8 cases: mutations of
    fp8_partials in mut)."""
    c = gc.case
    if gc.a8:
        S = tc_split(c, sms, int(gc.env.get("B2_GEMM_TC_MAX_SPLIT", TC_MAX_SPLIT)))
        return restate_fp8(c, inp["wt"], inp["A"], S, gc.act, gc.alpha, inp["bias"], inp["res"], inp["wt2"], **mut)
    W = path_weights(c, inp["wt"], gc.path) if W is None else W
    if c.pair:
        W2 = path_weights(c, inp["wt2"], gc.path) if W2 is None else W2
        return expected(inp["A"], W, alpha=gc.alpha, W2=W2)
    return expected(inp["A"], W, gc.act, gc.alpha, inp["bias"], inp["res"], **mut)


def case_precondition(gc, inp):
    if gc.a8:
        return precondition_fp8(gc.case, inp["wt"], inp["A"], inp["wt2"])
    return precondition(gc.case, inp["wt"], inp["A"], gc.path, gc.alpha, inp["bias"], inp["res"], gc.act,
                        unit_a=2.0 ** -gc.e, W2wt=inp["wt2"])


# fp8 activations x int4 per-channel weights (b2_gemm_wq_run_fp8): M 1, 17, 64, K with an odd number of 64-k tiles, split-K,
# MULTI, SwiGLU pair; and the read-back (one-hot rows: code 448 times the weight code, scale fp32(1/448))
FP8_CASES = [
    _gc("fp8-m1", Case(4, 1088, 130), 1, "tc8", bias=True, res=True),
    _gc("fp8-m17-silu", Case(4, 3648, 640), 17, "tc8", act=ACT_SILU, alpha=0.5, res=True),
    _gc("fp8-m64", Case(4, 3584, 4608), 64, "tc8", bias=True, res=True),
    _gc("fp8-m64-multi-gelu", Case(4, 1088, 18944), 64, "tc8", act=ACT_GELU_ERF),
    _gc("fp8-m40-relu", Case(4, 1088, 1290), 40, "tc8", act=ACT_RELU, bias=True, alpha=0.5),
    _gc("fp8-pair", Case(4, 1088, 704, pair=True), 20, "tc8"),
    _gc("rb-fp8-m64", Case(4, 1088, 130), 64, "tc8"),
    _gc("rb-fp8-m17", Case(4, 1088, 130), 17, "tc8"),
]
