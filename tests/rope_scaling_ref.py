"""Independent fp64 restatements of the scaled-rotary frequency tables (ops.rope_table), a restatement of the table form's
fp32 arithmetic (b2_rope_table in include/b200spark.h) with its error bound, and a decode-stack oracle that rotates with the
table.

Tables.  inv_ref restates the published Hugging Face definitions one frequency at a time with Python floats (no tensors, no
shared code with ops.rope_table), so the two agree to the final fp32 rounding.

Kernel.  For a q or k head row x (FT values), rotary position pos and a table row inv (fp32), per dim d < rotary_dim with
f = d % half and partner p = -x[d + half] (d < half) or x[d - half]:
    ang = fl32(pos inv[f]);  cs, sn = sincosf(ang) (2 ulp);  c = fl32(cs af);  s = fl32(sn af);
    y = FT(fl32(fma(x, c, fl32(p s)))).
Against Y = x af cos(ang) + p af sin(ang) in fp64 at the same fp32 angle, the error before the FT rounding is at most
    af (|x| + |p|) (2^-23 + 3 * 2^-24) < D = af (|x| + |p|) 2^-21
(sincosf's 2 ulp below 1 is 2^-23, then the af products, the partner product and the fma each round once), so
    |y - Y| <= ulp_FT(|Y| + D) / 2 + D      (glue_ref.rope_ratio).
The angle needs no slack: it is fl32(pos inv[f]) on the host and the device alike.  Dims >= rotary_dim and V rows keep
their bits."""
import math

import numpy as np
import torch

import glue_ref as G
import qk_norm_ref as QR

HEAD = 128
# the wrong kernels the bound must reject by >= 4x (tests/test_rope_scaling_cpu.py)
BUGS = ["neighbour_row", "freq_shift", "af_q_only", "af_twice", "slot_pos"]

QWEN25 = (1e6, {"rope_type": "yarn", "factor": 4.0, "original_max_position_embeddings": 32768})
QWEN3 = (1e6, {"type": "yarn", "factor": 4.0, "original_max_position_embeddings": 32768})  # legacy "type" key
LLAMA31 = (5e5, {"rope_type": "llama3", "factor": 8.0, "low_freq_factor": 1.0, "high_freq_factor": 4.0,
                 "original_max_position_embeddings": 8192})
LINEAR = (1e4, {"rope_type": "linear", "factor": 2.0})
# YaRN over a small native context (256), for the CPU table tests: the correction dims are 1 and 18 at rotary_dim 128 (0 and
# 9 at 64), so the ramp sits at the start of the table and most frequencies are interpolated, unlike the Qwen2.5 entry
# (23 and 40)
TINY_YARN = (1e6, {"rope_type": "yarn", "factor": 4.0, "original_max_position_embeddings": 256})


def inv_ref(scaling, base, d):
    """(fp32 inverse frequencies [d / 2], attn_factor) restated per frequency in Python floats"""
    kind = "default" if not scaling else scaling.get("rope_type", scaling.get("type"))
    out, af = [], 1.0
    for f in range(d // 2):
        theta = 1.0 / (base ** (2.0 * f / d))
        if kind == "default":
            v = theta
        elif kind == "linear":
            v = theta / scaling["factor"]
        elif kind == "yarn":
            s, L = scaling["factor"], scaling["original_max_position_embeddings"]
            dim_of = lambda rot: d * math.log(L / (rot * 2.0 * math.pi)) / (2.0 * math.log(base))
            lo = max(math.floor(dim_of(scaling.get("beta_fast", 32))), 0)
            hi = min(math.ceil(dim_of(scaling.get("beta_slow", 1))), d - 1)
            if hi == lo:
                hi += 0.001
            ramp = min(max((f - lo) / (hi - lo), 0.0), 1.0)
            v = theta / s * ramp + theta * (1.0 - ramp)
            af = scaling.get("attention_factor") or (0.1 * math.log(s) + 1.0 if s > 1 else 1.0)
        elif kind == "llama3":
            s, L = scaling["factor"], scaling["original_max_position_embeddings"]
            a, c = scaling["low_freq_factor"], scaling["high_freq_factor"]
            wl = 2.0 * math.pi / theta
            if wl < L / c:
                v = theta
            elif wl > L / a:
                v = theta / s
            else:
                g = (L / wl - a) / (c - a)
                v = (1.0 - g) * theta / s + g * theta
        else:
            raise ValueError(kind)
        out.append(v)
    return np.array(out, np.float64).astype(np.float32), af


def yarn_dims(scaling, base, d):
    """(low, high) correction dims of a YaRN entry"""
    L = scaling["original_max_position_embeddings"]
    dim_of = lambda rot: d * math.log(L / (rot * 2.0 * math.pi)) / (2.0 * math.log(base))
    return max(math.floor(dim_of(32)), 0), min(math.ceil(dim_of(1)), d - 1)


def _partner(x, rd):
    half = rd // 2
    a = x[..., :rd]
    return np.concatenate([-a[..., half:], a[..., :half]], -1)


def _setup(x, pos, inv, af, n_heads, rd, seq, slots, bug):
    """per-element angle (fp32), amplitude factor and partner for rows x [R, heads, 128]"""
    x = np.asarray(x, np.float32)
    R, heads = x.shape[:2]
    inv = np.asarray(inv, np.float32).reshape(-1, np.asarray(inv).shape[-1])
    seq = np.zeros(R, int) if seq is None else np.asarray(seq)
    row = seq % inv.shape[0]
    if bug == "neighbour_row":
        row = (seq + 1) % inv.shape[0]
    tab = inv[row][:, :rd // 2]
    if bug == "freq_shift":
        tab = np.concatenate([tab[:, 1:], tab[:, -1:]], -1)
    tab = np.concatenate([tab, tab], -1)                           # [R, rd]: f = d % half
    p = np.asarray(slots if bug == "slot_pos" else pos)
    ang = (p.astype(np.float32)[:, None] * tab).astype(np.float32)  # [R, rd]
    amp = np.full((R, heads, 1), af, np.float64)
    if bug == "af_q_only":
        amp[:, n_heads:] = 1.0
    if bug == "af_twice":
        amp = amp * af
    return x, ang[:, None, :], amp, _partner(x, rd)


def table_formula(x, pos, inv, af, n_heads, rd, seq=None, slots=None, bug=None):
    """(Y, D) of the bound above for q and k rows x [R, heads, 128] (heads [0, n_heads) q, the rest k), positions pos [R],
    table rows inv [S, >= rd / 2] (S = 1: shared; else row seq[r] for row r); bug: one of BUGS (slots: the rows' slots)"""
    x, ang, amp, o = _setup(x, pos, inv, af, n_heads, rd, seq, slots, bug)
    a = x[..., :rd].astype(np.float64)
    o = o.astype(np.float64)
    ang = ang.astype(np.float64)
    Y = x.astype(np.float64).copy()
    Y[..., :rd] = a * amp * np.cos(ang) + o * amp * np.sin(ang)
    D = np.zeros_like(Y)
    D[..., :rd] = np.abs(amp) * (np.abs(a) + np.abs(o)) * 2.0 ** -21
    return Y, D


def table_kernel32(x, pos, inv, af, n_heads, rd, dt, seq=None):
    """the kernel's arithmetic in numpy fp32 (cos / sin of the fp32 angle correctly rounded), rounded once to FT, as fp64"""
    x, ang, amp, o = _setup(x, pos, inv, af, n_heads, rd, seq, None, None)
    f32 = np.float32
    cs, sn = np.cos(ang.astype(np.float64)).astype(f32), np.sin(ang.astype(np.float64)).astype(f32)
    c, s = (cs * amp.astype(f32)).astype(f32), (sn * amp.astype(f32)).astype(f32)
    t = (o * s).astype(f32)
    y = x.astype(np.float64).copy()
    y[..., :rd] = (x[..., :rd].astype(np.float64) * c + t).astype(f32)
    return G.rn(y, dt)


def ratio(y, Y, D, dt):
    return G.rope_ratio(y, Y, D, dt)


# ------------------------------------------------------------------------------------------------ decode-stack oracle
def ref_from_stack(stack, kv_mode, exact=False):
    """the oracle of the stack (with the per-head Q/K norm when its layers carry one) whose rotary uses the stack's
    frequency table in fp64: ang = pos inv_f, cos and sin scaled by attn_factor, rounded to fp32 like the base oracle's"""
    ref = QR.ref_from_stack(stack, kv_mode, exact=exact)
    if stack.cfg.rope_scaling is not None:
        inv, af = stack.rope
        base_cls = ref.__class__
        ref.__class__ = type("Table" + base_cls.__name__, (TableRopeMixin, base_cls), {})
        ref.rope_inv, ref.rope_af = inv.double().cpu(), float(af)
    return ref


class TableRopeMixin:
    def _rope(self, x, pos):
        half = x.shape[-1] // 2
        ang = pos * self.rope_inv[:half]
        cs, sn = (torch.cos(ang) * self.rope_af).float(), (torch.sin(ang) * self.rope_af).float()
        a, b = x[:, :half], x[:, half:]
        return torch.cat([a * cs - b * sn, b * cs + a * sn], dim=-1)
