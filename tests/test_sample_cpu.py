"""CPU: the restatement of b2_sample (tests/sample_ref.py) and the library's argument checks, without a GPU.

Philox4x32-10 reproduces Random123's known-answer vectors; each restated bug of MUTATIONS changes a drawn id on the
constructed cases; bad arguments return B2_ERR_PARAM / B2_ERR_LIMIT before any launch."""
import numpy as np
import pytest
import torch

import sample_ref as S

B2_ERR_PARAM, B2_ERR_LIMIT = 3, 4


@pytest.mark.parametrize("ctr,key,want", [
    ((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
    ((0xffffffff,) * 4, (0xffffffff,) * 2, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
    ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0), (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1)),
])
def test_philox_known_answers(ctr, key, want):
    assert tuple(int(v) for v in S.philox(ctr, key)) == want


def test_exact_rows_have_power_of_two_weights():
    rng = np.random.default_rng(0)
    for j in (0, 1, 3):
        x = S.exact_row(4097, j, 0.0 if j else 2.0, rng, torch.bfloat16, neg_inf=3)
        plan = S.row_plan(x, S.exact_temperature(j), 0, 1.0)
        w = plan["w"]
        assert w[0] == S.TWO40 and np.all((w == 0) | ((w & (w - 1)) == 0))


def _cases():
    """(x, t, k, p, seed, off, row): small rows with ties at the boundaries, +-0 and zero-weight tails"""
    t1 = S.exact_temperature(0)  # c = 1
    tie = np.array([0, -1, -1, -1, -2, -2, -3, -5, -60], np.float32)  # weights 2^40, 2^39 x3, 2^38 x2, 2^37, 2^35, 0
    zeros = np.array([-0.0, 0.0, -1, -0.0, -2], np.float32)
    half = np.array([0, -1, -1], np.float32)  # S = 2^41: at p = 0.5 the maximum alone reaches Pt exactly
    cases = []
    for seed in range(4):
        for off in range(16):
            for k, p in ((0, 1.0), (2, 1.0), (3, 1.0), (0, 0.5), (0, 0.6), (0, 0.75), (4, 0.9)):
                cases.append((tie, t1, k, p, seed, off, 3))
                cases.append((zeros, t1, k, p, seed, off, 5))
                cases.append((half, t1, k, p, seed, off, 2))
                cases.append((tie[::-1].copy(), S.exact_temperature(1), k, p, seed, off, 1))
    return cases


@pytest.mark.parametrize("variant", S.MUTATIONS)
def test_mutations_change_a_drawn_id(variant):
    """every restated bug draws another id on at least one constructed case"""
    changed = 0
    for x, t, k, p, seed, off, row in _cases():
        a = S.sample_row(x, t, k, p, seed, off, row)
        try:
            b = S.sample_row(x, t, k, p, seed, off, row, variant=variant)
        except AssertionError:  # the variant's weights are no longer exact: a different row plan, a different draw
            b = -1
        changed += a != b
    assert changed > 0, variant


def test_greedy_rows_and_uniform_temperature():
    x = np.array([1.0, 3.0, 3.0, -np.inf, 2.0], np.float32)
    for t in (0.0, -1.0, np.nan, 2.0 ** -130):
        assert S.sample_row(x, t, 0, 1.0, 7, 0) == 1
    assert S.sample_row(np.array([1.0, np.nan, np.inf], np.float32), 1.0, 0, 1.0, 7, 0) == 1
    assert S.sample_row(np.full(4, -np.inf, np.float32), 1.0, 0, 1.0, 7, 0) == 0
    plan = S.row_plan(x, np.inf, 0, 1.0)  # c = 0: every finite entry weighs 2^40, -inf nothing
    assert list(plan["w"]) == [S.TWO40] * 4 + [0]
    assert S.sample_row(x, 1.0, 1, 1.0, 7, 0, form="fp64") == 1 and S.sample_row(x, 1.0, 0, 0.0, 7, 0, form="fp64") == 1


def test_draw_counts_of_a_row():
    """the histogram of 4096 draws over consecutive offsets follows the weights (exact row, no filter)"""
    x = np.array([0, -1, -1, -2, -3, -50], np.float32)
    plan = S.row_plan(x, S.exact_temperature(0), 0, 1.0)
    ids = S.draw(plan, S.draw_u24(11, np.arange(4096, dtype=np.uint64)))
    h = np.bincount(ids, minlength=6)
    assert h[5] == 0 and h[0] > h[1] > h[3] > h[4] > 0 and abs(h[1] - h[2]) < 200


def test_argument_checks_without_gpu():
    """every rejected call returns before a launch (the addresses are never dereferenced)"""
    from b200spark import _lib
    lib, bf = _lib.lib, _lib.DT_BF16
    A = 1 << 20
    ok = [A, A, 1, 100, 100, A, A, A, A, A, bf]
    for i in (0, 1, 5, 6, 7, 8, 9):  # each pointer NULL
        a = list(ok)
        a[i] = None
        assert lib.b2_sample(*a, None) == B2_ERR_PARAM, i
    for i, v in ((2, -1), (3, 0), (4, 99), (10, _lib.DT_F32), (10, _lib.DT_I8)):
        a = list(ok)
        a[i] = v
        assert lib.b2_sample(*a, None) == B2_ERR_PARAM, (i, v)
    a = list(ok)
    a[3], a[4] = _lib.SAMPLE_MAX_N + 1, _lib.SAMPLE_MAX_N + 1
    assert lib.b2_sample(*a, None) == B2_ERR_LIMIT
    a = list(ok)
    a[2] = 0
    assert lib.b2_sample(*a, None) == 0  # no rows: nothing to launch


def test_decode_stack_sampling_limits():
    from b200spark import model
    with pytest.raises(AssertionError, match="q_len == 1"):
        model.DecodeStack(model.TINY, 1, 16, q_len=4, sample=True, device="cpu")
    with pytest.raises(AssertionError, match="tp_size == 1"):
        model.DecodeStack(model.TINY, 1, 16, tp_size=2, sample=True, device="cpu")
