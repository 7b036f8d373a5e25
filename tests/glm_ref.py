"""GLM rotary references: the reference's interleaved ("half_inner") rotary restated, its two inverse-frequency formulas, an
fp64 Hugging Face-style GLM rotary, the dim permutation P that maps the interleaved pairing onto NeoX, and a decode-stack
oracle that rotates the way a GLM stack does.

Reference semantics (ChatGLM2 / ChatGLM3 / GLM-4: RotaryMulQuery with rotary_type 3).  Of each q and k head of 128 dims
only the first 64 rotate, in pairs (x[2i], x[2i+1]) at frequency i < 32; dims 64 .. 127 pass through.  With the fp32
frequency inv[i] and position pos:
    ang = fl32(inv[i] pos);  c, s = cos(ang), sin(ang) in fp32;
    y[2i] = FT(fl32(x[2i] c) - fl32(x[2i+1] s)),  y[2i+1] = FT(fl32(x[2i+1] c) + fl32(x[2i] s)).
Inverse frequencies over rotary_dim = head / 2 = 64, rounded once to fp32:
    invfreq_type 1 (ChatGLM2):          inv_i = base^(-2i / 64) / rope_ratio;
    invfreq_type 2 (ChatGLM3, GLM-4):   inv_i = (base rope_ratio)^(-2i / 64).
Bound.  Against the fp64 rotary at theta_i (the same formula without any rounding) the restatement and the library's
kernels meet glue_ref's NeoX bound: the pairing only decides which dim is the partner, and the angle error is at most
pos theta (2^-22 + 2^-24 + ...) <= pos 2^-21 as there (theta <= 1), so per element
    |y - Y64| <= ulp_FT(|Y64| + D64) / 2 + D64,   D64 = (|x| + |partner|) (2^-22 + pos 2^-21).

Permutation.  P de-interleaves the first rotary_dim dims of a head (evens, then odds) and keeps the rest.  The library's
interleaved rotary runs the NeoX instructions on the pair (2i, 2i + 1) that NeoX runs on (i, i + rotary_dim / 2), so
    interleaved(x) = P^-1 neox(P x), bit for bit."""
import numpy as np
import torch

import glue_ref as G
import qk_norm_ref as QR

HEAD = 128


# ------------------------------------------------------------------------------------------------ frequencies
def invfreq(invfreq_type, base, rope_ratio, rotary_dim=64):
    """fp32 [rotary_dim / 2] inverse frequencies of the reference's invfreq_type 1 or 2, from fp64"""
    i = np.arange(rotary_dim // 2, dtype=np.float64)
    if invfreq_type == 1:
        v = np.float64(base) ** (-2.0 * i / rotary_dim) / np.float64(rope_ratio)
    elif invfreq_type == 2:
        v = (np.float64(base) * np.float64(rope_ratio)) ** (-2.0 * i / rotary_dim)
    else:
        raise ValueError(invfreq_type)
    return v.astype(np.float32)


def theta64(invfreq_type, base, rope_ratio, rotary_dim=64):
    """the same frequencies in fp64 (the Hugging Face GLM rotary's, with rope_ratio folded in)"""
    i = np.arange(rotary_dim // 2, dtype=np.float64)
    if invfreq_type == 1:
        return np.float64(base) ** (-2.0 * i / rotary_dim) / np.float64(rope_ratio)
    return (np.float64(base) * np.float64(rope_ratio)) ** (-2.0 * i / rotary_dim)


# ------------------------------------------------------------------------------------------------ permutation
def perm(rotary_dim, head=HEAD):
    """index array of P: (P x)[k] = x[perm[k]]"""
    return np.concatenate([np.arange(0, rotary_dim, 2), np.arange(1, rotary_dim, 2), np.arange(rotary_dim, head)])


def apply_p(x, rotary_dim):
    return x[..., perm(rotary_dim, x.shape[-1])]


def apply_p_inv(y, rotary_dim):
    out = np.empty_like(y) if isinstance(y, np.ndarray) else torch.empty_like(y)
    out[..., perm(rotary_dim, y.shape[-1])] = y
    return out


def _pair_partner(x, rotary_dim):
    """interleaved partner of each rotated dim: -x[d + 1] for even d, x[d - 1] for odd d"""
    a = x[..., :rotary_dim]
    o = np.empty_like(a)
    o[..., 0::2] = -a[..., 1::2]
    o[..., 1::2] = a[..., 0::2]
    return o


# ------------------------------------------------------------------------------------------------ rotaries
def half_inner32(x, pos, inv, dt):
    """the reference's half_inner kernel restated in numpy fp32 (cos / sin of the fp32 angle correctly rounded to fp32),
    rounded once to dt.  x [..., head] FT values, pos [...] (one position per row), inv fp32 [head / 4]."""
    x = np.asarray(x, np.float32)
    f32 = np.float32
    inv = np.asarray(inv, f32)
    ang = (inv * np.asarray(pos)[..., None].astype(f32)).astype(f32)         # [..., 32]
    c, s = np.cos(ang.astype(np.float64)).astype(f32), np.sin(ang.astype(np.float64)).astype(f32)
    v1, v2 = x[..., 0:2 * inv.shape[-1]:2], x[..., 1:2 * inv.shape[-1]:2]
    y = x.astype(np.float64).copy()
    y[..., 0:2 * inv.shape[-1]:2] = ((v1 * c).astype(f32) - (v2 * s).astype(f32)).astype(f32)
    y[..., 1:2 * inv.shape[-1]:2] = ((v2 * c).astype(f32) + (v1 * s).astype(f32)).astype(f32)
    return G.rn(y, dt)


def glm64(x, pos, theta, rotary_dim):
    """fp64 Hugging Face-style GLM rotary (pairs (2i, 2i+1) at theta[i]) and the slack D64 of the bound"""
    x = np.asarray(x, np.float64)
    pos = np.asarray(pos, np.float64)[..., None]
    th = np.repeat(np.asarray(theta, np.float64), 2)                          # [rotary_dim]: f = d / 2
    a, o = x[..., :rotary_dim], _pair_partner(x, rotary_dim)
    Y = x.copy()
    Y[..., :rotary_dim] = a * np.cos(pos * th) + o * np.sin(pos * th)
    D = np.zeros_like(Y)
    D[..., :rotary_dim] = (np.abs(a) + np.abs(o)) * (2.0 ** -22 + pos * 2.0 ** -21)
    return Y, D


def il_kernel32(x, pos, base, rotary_dim, dt):
    """the library's computed-frequency interleaved rotary written pair by pair (f = d / 2, partner d ^ 1) in numpy fp32,
    with the frequencies of its NeoX form (glue_ref.rope_tables), rounded once to dt"""
    x = np.asarray(x, np.float32)
    f, z, inv = G.rope_tables(base, rotary_dim)
    inv_f = inv[:rotary_dim // 2]                                            # inv depends on f only
    ang = (np.asarray(pos)[..., None].astype(np.float32) * np.repeat(inv_f, 2)).astype(np.float32)
    cs, sn = np.cos(ang.astype(np.float64)).astype(np.float32), np.sin(ang.astype(np.float64)).astype(np.float32)
    y = x.copy()
    y[..., :rotary_dim] = x[..., :rotary_dim] * cs + _pair_partner(x, rotary_dim) * sn
    return G.ft_values(y, dt)


def il_formula(x, pos, base, rotary_dim):
    """(Y, D) of glue_ref.rope_formula for the interleaved pairing: the NeoX formula on P x, permuted back"""
    Y, D = G.rope_formula(apply_p(np.asarray(x, np.float32), rotary_dim), pos, base, rotary_dim)
    return apply_p_inv(Y, rotary_dim), apply_p_inv(D, rotary_dim)


# ------------------------------------------------------------------------------------------------ decode-stack oracle
def ref_from_stack(stack, kv_mode, exact=False):
    """the oracle of a stack (with the Q/K norm when its layers carry one) whose rotary covers cfg.rotary_dim dims with the
    cfg.rope_style pairing: fp64 angles, cos and sin rounded to fp32, fp32 products (as the base oracle's NeoX rotary)"""
    ref = QR.ref_from_stack(stack, kv_mode, exact=exact)
    cfg = stack.cfg
    if cfg.rotary_dim is not None or cfg.rope_style != "neox":
        base_cls = ref.__class__
        ref.__class__ = type("Glm" + base_cls.__name__, (GlmRopeMixin, base_cls), {})
        rd = cfg.rotary_dim or stack.head
        if cfg.rope_scaling is not None:
            ref.rope_theta, ref.rope_af = stack.rope[0].double().cpu(), float(stack.rope[1])
        else:
            ref.rope_theta = torch.tensor(cfg.rope_base, dtype=torch.float64) ** (
                -torch.arange(0, rd // 2, dtype=torch.float64) * 2.0 / float(rd))
            ref.rope_af = 1.0
        ref.rope_dim, ref.rope_il = rd, cfg.rope_style == "interleaved"
    return ref


class GlmRopeMixin:
    def _rope(self, x, pos):
        rd = self.rope_dim
        ang = pos * self.rope_theta
        cs, sn = (torch.cos(ang) * self.rope_af).float(), (torch.sin(ang) * self.rope_af).float()
        out = x.clone()
        if self.rope_il:
            a, b = x[:, 0:rd:2], x[:, 1:rd:2]
            out[:, 0:rd:2] = a * cs - b * sn
            out[:, 1:rd:2] = b * cs + a * sn
        else:
            a, b = x[:, :rd // 2], x[:, rd // 2:rd]
            out[:, :rd] = torch.cat([a * cs - b * sn, b * cs + a * sn], dim=-1)
        return out
