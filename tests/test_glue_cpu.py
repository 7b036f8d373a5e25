"""CPU: the bounds of tests/glue_ref.py are sharp (the numpy restatement of each kernel formula passes them, known-wrong
variants fail them), the argmax order is the one the kernels implement, and the glue ops' argument checks reject bad
arguments before any device work."""
import ctypes as C

import numpy as np
import pytest
import torch

import glue_ref as G


@pytest.mark.parametrize("dt", ["bf16", "fp16"])
def test_rmsnorm_restatement_within_bound(dt):
    """every row kind, every width: the fp32 restatement is within the bound and rarely off rn_FT(exact)"""
    ft = G.FTS[dt]
    for cols in G.RMS_COLS:
        for eps in G.RMS_EPS:
            x, g = G.rms_batch(12, cols, ft, seed=cols)
            y = G.ft_values(G.rms_kernel32(x, g, eps), ft)
            ratio, miss, n = G.rms_check(y, x, g, eps, ft)
            assert ratio <= 1.0, (cols, eps, ratio)
            assert miss <= G.rms_allowed_mismatches(n), (cols, eps, miss)
        print("cols %5d: sum depth %3d, eps_rms = %.1f u = %.3g" % (cols, G.rms_depth(cols), G.rms_eps(cols) / G.U32, G.rms_eps(cols)))


@pytest.mark.parametrize("variant,kind", [("eps_outside", "tiny"), ("sum", "random"), ("sum", "constant")])
def test_rmsnorm_wrong_variants_rejected(variant, kind):
    rng = np.random.default_rng(3)
    for dt in G.FTS.values():
        x = G.rms_rows(kind, 4, 896, dt, rng)
        g = G.rms_gamma(896, dt, rng)
        ratio, _, _ = G.rms_check(G.ft_values(G.rms_kernel32(x, g, 1e-5, variant=variant), dt), x, g, 1e-5, dt)
        assert ratio > 1.0, (variant, kind, ratio)


def test_rmsnorm_bound_is_tight():
    """the bound is within a hair of half an ulp: rn(exact) moved one ulp away from exact is rejected everywhere"""
    x, g = G.rms_batch(6, 3584, torch.bfloat16, seed=1)
    ex = G.rms_exact(x, g, 1e-6)
    r = G.rn(ex, torch.bfloat16)
    off = np.abs(ex) > 0
    bumped = r - np.where(ex >= r, 1.0, -1.0) * G.ulp(r, torch.bfloat16)
    ratio = np.abs(bumped - ex) / (G.ulp(ex, torch.bfloat16) / 2 + G.rms_eps(3584) * np.abs(ex))
    assert np.all(ratio[off] > 1.0)


def _rope_inputs(rotary_dim, dt, seed):
    rng = np.random.default_rng(seed)
    x = G.ft_values(rng.standard_normal((len(G.ROPE_POS), 3, 128)) * 2, dt)
    return x, np.array(G.ROPE_POS)[:, None]  # pos broadcast over the 3 heads


@pytest.mark.parametrize("rotary_dim", [128, 64, 32])
@pytest.mark.parametrize("dt", ["bf16", "fp16"])
def test_rope_restatement_within_bounds(rotary_dim, dt):
    """the fp32 restatement passes both bounds at every position and base; dims >= rotary_dim are untouched"""
    ft = G.FTS[dt]
    x, pos = _rope_inputs(rotary_dim, ft, rotary_dim)
    for base in G.ROPE_BASES:
        y = G.rope_kernel32(x, pos, base, rotary_dim, ft)
        Y, D = G.rope_formula(x, pos, base, rotary_dim)
        assert G.rope_ratio(y, Y, D, ft).max() <= 1.0, base
        Y64, D64 = G.rope_neox64(x, pos, base, rotary_dim)
        assert G.rope_ratio(y, Y64, D64, ft).max() <= 1.0, base
        assert np.array_equal(y[..., rotary_dim:], x[..., rotary_dim:])


@pytest.mark.parametrize("wrong", ["partner", "sign", "pos"])
@pytest.mark.parametrize("rotary_dim", [128, 64])
def test_rope_wrong_variants_rejected(wrong, rotary_dim):
    """the wrong rotate-half partner and the wrong sign fail the formula bound at every position but 0 (where sin = 0
    hides the partner), a position off by one at every position (one step of angle is a whole radian in dim 0)"""
    ft = torch.bfloat16
    x, pos = _rope_inputs(rotary_dim, ft, 7)
    for base in G.ROPE_BASES:
        y = G.rope_kernel32(x, pos, base, rotary_dim, ft)
        Y, D = G.rope_formula(x, pos, base, rotary_dim, wrong=wrong)
        worst = G.rope_ratio(y, Y, D, ft).reshape(len(G.ROPE_POS), -1).max(1)
        assert np.all(worst[0 if wrong == "pos" else 1:] > 1.0), (wrong, base, worst)


def test_rope_neox_bound_grows_with_position():
    """the fp64 slack is position-only: 2^-22 at 0, 2^-21 pos beyond; the formula slack is 0 in dim 0 (inv = 1 exactly)"""
    x = np.ones((2, 128), np.float32)
    _, D64 = G.rope_neox64(x, np.array([0, 131071]), 1e6, 128)
    assert np.allclose(D64[0, :128], 2 * 2.0 ** -22) and np.allclose(D64[1, :128], 2 * (2.0 ** -22 + 131071 * 2.0 ** -21))
    _, D = G.rope_formula(x, np.array([131071]), 1e6, 128)
    assert D[0, 0] == 2 * 2.0 ** -22 and D[0, 1] > D[0, 0]


@pytest.mark.parametrize("n", G.ARGMAX_N)
def test_argmax_blocked_restatement_is_np_argmax(n):
    """the kernel's reduction with its order equals np.argmax on every row kind (ids and values); ties resolved to the
    highest index fail on the tie kinds; before NaN was ordered, an all-NaN row gave index INT_MAX"""
    x = G.argmax_batch(n, len(G.ARGMAX_KINDS), 0, seed=n)
    ids, vals = G.argmax_ref(x, n)
    wrong = 0
    for r, kind in enumerate(G.ARGMAX_KINDS):
        i, v = G.argmax_blocked(x[r, :n])
        assert i == ids[r] and (v == vals[r] or (np.isnan(v) and np.isnan(vals[r]))), (kind, i, ids[r])
        if kind in G.TIE_PLANTS or kind in ("first_last", "equal"):
            wrong += G.argmax_blocked(x[r, :n], G.beats_highest_tie)[0] != ids[r]
        if kind == "nan_all":
            assert G.argmax_blocked(x[r, :n], G.beats_before_nan_fix)[0] == 0x7FFFFFFF
    if n > 1:  # one element cannot tie
        assert wrong >= 2


def test_tie_plants_hit_their_reduction_step():
    """each planted pair is decided where its name says: one thread (same i % 1024), one warp (same (i % 1024) // 32),
    different warps"""
    th = {k: [i % 1024 for i in v] for k, v in G.TIE_PLANTS.items()}
    assert th["tie_stride"][0] == th["tie_stride"][1]
    assert th["tie_lanes"][0] != th["tie_lanes"][1] and th["tie_lanes"][0] // 32 == th["tie_lanes"][1] // 32
    for k in ("tie_warps", "tie_final"):
        assert th[k][0] // 32 != th[k][1] // 32
    assert (th["tie_final"][0] // 32) ^ (th["tie_final"][1] // 32) >= 16  # decided at the widest butterfly step


@pytest.mark.parametrize("tp", [2, 4, 8])
def test_shard_merge_restatement(tp):
    """argmax of each shard + the merge == argmax of the whole row, for every hard kind; ties across shards and NaN in
    two shards go to the lowest rank"""
    rng = np.random.default_rng(tp)
    n = 152064
    for kind in G.TP_KINDS:
        x = G.tp_row(kind, n, tp, rng)
        pairs = [G.argmax_blocked(x[s:e]) for s, e in G.shard_bounds(n, tp)]
        ids = np.array([[i + s] for (i, _), (s, _) in zip(pairs, G.shard_bounds(n, tp))])
        vals = np.array([[v] for _, v in pairs], np.float32)
        assert G.merge_ref(vals, ids)[0] == np.argmax(x), kind
        if kind in ("tie_shards", "tie_all_shards"):  # a merge that lets a later rank win ties is wrong here
            assert G.merge_ref(vals, ids, lambda v, i, best, bi: v >= best)[0] != np.argmax(x), kind
        if kind == "nan_shards":  # and so is one that compares NaN like a number
            assert G.merge_ref(vals, ids, G.beats_before_nan_fix)[0] != np.argmax(x)


def test_binary_reference_overflows_in_fp16():
    a = torch.tensor([60000.0, -60000.0, 300.0, 1.0], dtype=torch.float16)
    b = torch.tensor([60000.0, -60000.0, 300.0, 2.0 ** -24], dtype=torch.float16)
    s = G.binary_ref(a, b, True, torch.float16)
    m = G.binary_ref(a, b, False, torch.float16)
    assert s.tolist()[:2] == [float("inf"), float("-inf")] and m.tolist()[2] == float("inf")
    assert s.tolist()[3] == 1.0  # 1 + 2^-24 rounds to 1 (one rounding of the fp32 sum)


B2_ERR_PARAM, B2_ERR_UNSUPPORTED = 3, 6


def test_rejected_arguments():
    """Misaligned vector pointers and ld < n are caught by the argument checks, before any device work (these calls
    never reach a launch, so the addresses are never dereferenced)."""
    from b200spark import _lib
    lib, bf, f16 = _lib.lib, _lib.DT_BF16, _lib.DT_F16
    A, M2, M8 = 1 << 20, (1 << 20) + 2, (1 << 20) + 8  # 16-byte aligned, 2 off, 8 off
    for ft in (bf, f16):
        for y, x, g in ((M2, A, A), (A, M8, A), (A, A, M2)):
            assert lib.b2_rmsnorm_ft(y, x, g, 1, 8, 1e-6, ft, None) == B2_ERR_UNSUPPORTED
        for o, a, b in ((M8, A, A), (A, M2, A), (A, A, M8)):
            assert lib.b2_binary_ft(o, a, b, 16, _lib.BIN_ADD, ft, None) == B2_ERR_UNSUPPORTED
        assert lib.b2_argmax_ft(A, None, A, 1, 100, 99, 0, ft, None) == B2_ERR_PARAM
    assert lib.b2_rmsnorm(M2, A, A, 1, 8, 1e-6, None) == B2_ERR_UNSUPPORTED
    assert lib.b2_binary(A, M2, A, 16, _lib.BIN_MUL, None) == B2_ERR_UNSUPPORTED
    assert lib.b2_embedding(M8, A, A, 1, 8, None) == B2_ERR_UNSUPPORTED
    assert lib.b2_embedding(A, M2, A, 1, 8, None) == B2_ERR_UNSUPPORTED
    rope = _lib.RopeCfg(1e6, 128, 0)
    assert lib.b2_rotary(A + 4, A, 1, 4, 2, 128, C.byref(rope), None) == B2_ERR_UNSUPPORTED
    assert lib.b2_rotary(A + 2, A, 1, 4, 2, 128, C.byref(rope), None) == B2_ERR_UNSUPPORTED
    assert lib.b2_argmax(A, A, 1, 100, 50, None) == B2_ERR_PARAM
    assert lib.b2_argmax_shard(A, A, A, 2, 100, 64, 0, None) == B2_ERR_PARAM


def test_python_dtype_guards():
    """b2_rotary and b2_argmax_shard are bf16 only: the wrappers refuse fp16 before calling the library"""
    from b200spark import ops
    with pytest.raises(TypeError):
        ops.rotary(torch.zeros(1, 8 * 128, dtype=torch.float16), torch.zeros(1, dtype=torch.int32), 4, 2)
    with pytest.raises(TypeError):
        ops.argmax_shard(torch.zeros(2, 64, dtype=torch.float16), 0, torch.zeros(2, dtype=torch.int64), torch.zeros(2))
