"""Restatement, exact-input candidates and error envelope of the per-head Q/K RMSNorm (QKLayerNormNoBeta): b2_qk_rmsnorm and
the fused form of b2_span_cache_append_qknorm (arithmetic: include/b200spark.h, b2_qk_norm).

Kernel.  One warp per 128-wide head row, 4 consecutive values per lane: ss = the lane's 4 squares added in order (squares of
16-bit values are exact in fp32), then an xor butterfly over 16, 8, 4, 2, 1; rs = rsqrtf(ss * 2^-7 + eps), with or without
an FMA; y = rn_FT(rn32(rn32(x rs) gamma)).

Exact inputs (x = j 2^-e with small integers j, dyadic gammas): ss and ss / 128 are exact, so the only freedom left is rs,
which lies within rsqrtf's 2 ulp of 1 / sqrt(t) for one of the two t forms.  Every row must equal the restatement bit for bit
for ONE of those candidates (norm_exact.rs_candidates), the same one for its 128 outputs.

Realistic rows.  Against exact = x gamma / sqrt(mean(x^2) + eps) in fp64, per element
    |y - exact| <= ulp_FT(exact) / 2 + QK_EPS |exact|
with QK_EPS derived as glue_ref.rms_eps derives its bound: the 8 additions of the sum (3 in the lane, 5 in the butterfly).

Fused form.  The append normalises a q or k row, rounds it to FT and applies the rotary of the append to that FT row; the
rotary contract of glue_ref (rope_formula / rope_ratio) holds against the restated FT norm output."""
import numpy as np
import torch

import glue_ref as G
import norm_exact as NE
from oracle import decoder_ref as DR

HEAD = 128
DEPTH = 3 + 5
QK_EPS = 1.01 * ((DEPTH + 2) / 2 + 4 + 2) * G.U32

# the wrong kernels the bounds must reject (each misses by >= 4 bounds on some case: tests/test_qk_norm_cpu.py)
BUGS = ["gamma_shift", "mean64", "eps_outside", "k_for_q", "v_normed", "after_rotary", "no_round"]


def sumsq(x):
    """fp32 sum of squares of [R, 128] rows in the kernel's order (lane sums, then the butterfly), as fp32 [R]"""
    x = np.asarray(x, np.float32).reshape(-1, 32, 4)
    s = x[:, :, 0] * x[:, :, 0]
    for i in range(1, 4):
        s = s + x[:, :, i] * x[:, :, i]
    for o in (16, 8, 4, 2, 1):
        s = s + s[:, np.arange(32) ^ o]
    return s[:, 0]


def head_norm(x, gamma, eps, dt, rs=None, bug=None, rounded=True):
    """restated kernel on [R, 128] rows (FT values as fp32) with gamma [128]; rs [R] overrides the nominal (correctly
    rounded, separate-multiply) rs.  Returns fp64 values (FT values unless rounded=False)."""
    x = np.asarray(x, np.float32)
    ss = sumsq(x).astype(np.float64)
    if rs is None:
        if bug == "mean64":
            rs = NE.rs_nominal(ss, 64, eps)
        elif bug == "eps_outside":
            rs = NE.f32(1.0 / (np.sqrt(NE.f32(ss / HEAD)) + NE.f32(eps)))
        else:
            rs = NE.rs_nominal(ss, HEAD, eps)
    g = np.asarray(gamma, np.float64)
    if bug == "gamma_shift":  # each lane reads the next lane's 4 gammas
        g = np.roll(g, -4)
    y = NE.f32(NE.f32(x.astype(np.float64) * np.asarray(rs)[:, None]) * g)
    return G.rn(y, dt) if rounded else y


def qk_rows(x, n_heads, n_groups, q_gamma, k_gamma, eps, dt, bug=None, rounded=True):
    """b2_qk_rmsnorm restated on [R, (nH + 2 nG) * 128] rows: q heads with q_gamma, k heads with k_gamma, V copied"""
    x = np.asarray(x, np.float32)
    R = x.shape[0]
    h = x.reshape(R, n_heads + 2 * n_groups, HEAD)
    y = h.astype(np.float64).copy()
    last = n_heads + (2 if bug == "v_normed" else 1) * n_groups
    for j in range(last):
        g = q_gamma if (j < n_heads and bug != "k_for_q") else k_gamma
        y[:, j] = head_norm(h[:, j], g, eps, dt, bug=bug, rounded=rounded)
    return y.reshape(R, -1)


def exact(x, n_heads, n_groups, q_gamma, k_gamma, eps):
    """fp64 QKLayerNormNoBeta of [R, (nH + 2 nG) * 128] rows (eps as the fp32 the kernel receives); V unchanged"""
    x = np.asarray(x, np.float64)
    R = x.shape[0]
    h = x.reshape(R, n_heads + 2 * n_groups, HEAD).copy()
    e = float(np.float32(eps))
    for j in range(n_heads + n_groups):
        g = np.asarray(q_gamma if j < n_heads else k_gamma, np.float64)
        h[:, j] = h[:, j] * g / np.sqrt(np.mean(h[:, j] ** 2, -1, keepdims=True) + e)
    return h.reshape(R, -1)


def ratio(y, ex, dt):
    """|y - exact| / (ulp_FT(exact) / 2 + QK_EPS |exact|) per element (V heads: exact = x, so any change shows)"""
    ex = np.asarray(ex, np.float64)
    return np.abs(np.asarray(y, np.float64) - ex) / (G.ulp(ex, dt) / 2 + QK_EPS * np.abs(ex))


def exact_rows_failing(y, x, gamma, eps, dt):
    """indices of the [R, 128] head rows y that match the restatement for NO rs candidate (same candidate for all 128)"""
    x = np.asarray(x, np.float32)
    cands, _ = NE.rs_candidates(sumsq(x).astype(np.float64), HEAD, eps)
    y = np.asarray(y, np.float64)
    ok = np.zeros(x.shape[0], bool)
    for c in range(cands.shape[1]):
        ok |= np.all(head_norm(x, gamma, eps, dt, rs=cands[:, c]) == y, axis=-1)
    return np.nonzero(~ok)[0]


def exact_batch(rows, dt, rng):
    """[rows, 128] x = j 2^-e (|j| <= 15, e per row in 0..8) and dyadic gammas k / 8 (k in 4..15): ss and ss / 128 exact"""
    j = rng.integers(-15, 16, (rows, HEAD)).astype(np.float64)
    e = rng.integers(0, 9, (rows, 1)).astype(np.float64)
    x = (j * 2.0 ** -e).astype(np.float32)
    return x, (rng.integers(4, 16, HEAD) / 8.0).astype(np.float32)


ROW_KINDS = ["normal", "spike"]


def realistic_rows(rows, width, dt, rng, kind, log2_rms):
    """[rows, width] FT values: N(0,1) rows or N(0,1) rows with one channel per head at 64 sigma, scaled to RMS 2^log2_rms"""
    x = rng.standard_normal((rows, width))
    if kind == "spike":
        h = x.reshape(rows, -1, HEAD)
        h[:, :, 7] = 64.0 * np.sign(h[:, :, 7] + 0.5)
    x = x * 2.0 ** log2_rms
    return G.ft_values(x, G.FTS[dt] if isinstance(dt, str) else dt)


def gammas(dt, rng):
    """(q_gamma, k_gamma) = 1 + 0.1 N(0,1) in FT, like the decode stack's"""
    return tuple(G.ft_values(1.0 + 0.1 * rng.standard_normal(HEAD), dt) for _ in range(2))


def rope_after(n, pos, base, rotary_dim):
    """rotary contract (glue_ref.rope_formula) of FT rows n [R, 128] at positions pos [R]"""
    return G.rope_formula(np.asarray(n, np.float32), pos, base, rotary_dim)


# ------------------------------------------------------------------------------------------------ decode-stack oracle
def ref_from_stack(stack, kv_mode, exact=False):
    """oracle.decoder_ref.from_stack with the per-head Q/K RMSNorm after the QKV GEMM and before rotary when the stack's
    layers carry qn / kn: fp32 math rounded to the model FT like every operator output (the reference's QKLayerNormNoBeta
    writes an FT tensor), no rounding with exact=True.  Layers without them are left as the base oracle runs them."""
    ref = DR.from_stack(stack, kv_mode, exact=exact)
    if stack.layers and "qn" in stack.layers[0]:
        ref.__class__ = QKNormRef
        ref.qk_gammas = {id(L["qkv"]): (S["qn"].float().cpu(), S["kn"].float().cpu()) for L, S in zip(ref.layers, stack.layers)}
    return ref


class QKNormRef(DR.RefDecoder):
    """RefDecoder whose QKV GEMM output passes through the per-head Q/K RMSNorm (qk_gammas: id of a layer's qkv weight ->
    (q_gamma, k_gamma) fp32)"""

    def _gemm(self, x, wb, act=None):
        y = super()._gemm(x, wb, act)
        g = self.qk_gammas.get(id(wb))
        if g is None:
            return y
        nH, nG = self.cfg.n_heads, self.cfg.n_kv
        h = y.float().reshape(y.shape[0], nH + 2 * nG, HEAD).clone()
        for sl, gm in ((slice(0, nH), g[0]), (slice(nH, nH + nG), g[1])):
            v = h[:, sl]
            h[:, sl] = v * torch.rsqrt(v.pow(2).mean(-1, keepdim=True) + self.cfg.eps) * gm
        return DR._bf(h.reshape(y.shape[0], -1))
