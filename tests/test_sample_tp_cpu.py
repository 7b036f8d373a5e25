"""CPU: the restatement of sampling under tensor parallelism (tests/sample_tp_ref.py) against b2_sample's
(tests/sample_ref.py), and the argument checks of b2_sample_shard / b2_sample_shard_merge, without a GPU.

For any contiguous split, P = 1 .. 8 ranks, unequal shards and single-column shards included, the protocol over records
draws b2_sample's id of the whole row; each restated bug of MUTATIONS draws another id on crafted rows (ties across
shard boundaries, a k-th element on a boundary, the nucleus ending on another rank than the draw)."""
import ctypes as C

import numpy as np
import pytest
import torch

import sample_ref as S
import sample_tp_ref as T

B2_ERR_PARAM, B2_ERR_LIMIT = 3, 4
KS = [0, 1, 2, 5, 50, -3]
PS = [1.0, 0.9, 0.5, 0.001, float("nan")]


@pytest.mark.parametrize("P", range(1, 9))
@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16])
def test_protocol_equals_whole_row_on_exact_rows(P, dt):
    rng = np.random.default_rng(100 * P + (dt == torch.float16))
    for it in range(24):
        n = int(rng.choice([P, P + 1, 37, 300, 1000, 4097]))
        j = int(rng.integers(0, 3))
        x = S.exact_row(n, j, 0.0 if it % 3 == 0 else 2.0, rng, dt, neg_inf=it % 4)
        t = S.exact_temperature(j)
        bounds = T.random_bounds(n, P, rng, one_col=it % 2 == 1) if it % 3 else T.even_bounds(n, P)
        k = int(rng.choice(KS + [n, n + 1]))
        p = float(rng.choice(PS))
        for off in range(6):
            seed = int(rng.integers(0, 2**63))
            want = S.sample_row(x, t, k, p, seed, off)
            got = T.shard_sample_row(x, bounds, t, k, p, seed, off, dt)
            assert got == want, (it, n, bounds, k, p, seed, off)


def test_greedy_and_non_finite_rows_take_the_whole_row_argmax():
    rng = np.random.default_rng(7)
    x = S.exact_row(97, 0, 1.0, rng, torch.bfloat16)
    for P in (2, 3, 8):
        b = T.random_bounds(97, P, rng)
        for t in (0.0, -1.0, float("nan"), 1e-45):  # t <= 0, NaN, c not finite
            assert T.shard_sample_row(x, b, t, 0, 1.0, 1, 2) == int(np.argmax(x))
        for v in (float("nan"), float("inf")):
            y = x.copy()
            y[[5, 60]] = v
            assert T.shard_sample_row(y, b, 1.0, 0, 1.0, 1, 2) == S.sample_row(y, 1.0, 0, 1.0, 1, 2) == 5
        y = np.full(97, -np.inf, np.float32)
        assert T.shard_sample_row(y, b, 1.0, 0, 1.0, 1, 2) == 0


def _crafted():
    """(x, bounds): rows of small integers at c = 1 (weights 2^(40 + x)) whose runs of equal values straddle the shard
    boundaries, with shards of different maxima"""
    run = np.array([-3, -1, -1, -1, -1, -2, -1, -1, -1, 0, -1, -1, -2, -2, -1, -1], np.float32)
    flat = np.array([-1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1], np.float32)
    steps = np.array([0, -1, -2, -3, -4, -4, -4, -4, -5, -6, -5, -6], np.float32)
    return [(run, [0, 4, 9, 16]), (run, [0, 1, 2, 10, 16]), (run, [0, 8, 16]), (flat, [0, 3, 6, 9, 12]), (flat, [0, 5, 12]),
            (steps, [0, 2, 6, 12]), (steps, [0, 1, 5, 7, 12])]


@pytest.mark.parametrize("variant", T.MUTATIONS)
def test_mutations_change_a_drawn_id(variant):
    t1 = S.exact_temperature(0)
    changed = 0
    for x, b in _crafted():
        for k, p in ((0, 1.0), (3, 1.0), (4, 1.0), (5, 0.9), (0, 0.5), (0, 0.3), (6, 0.75)):
            for off in range(24):
                want = S.sample_row(x, t1, k, p, 5, off)
                assert T.shard_sample_row(x, b, t1, k, p, 5, off) == want
                try:
                    got = T.shard_sample_row(x, b, t1, k, p, 5, off, variant=variant)
                except (AssertionError, IndexError):  # the bug leaves no holder, or two
                    got = -1
                changed += got != want
    assert changed > 0, variant


def _lib():
    from b200spark import _lib
    return _lib.lib


def test_record_and_state_sizes():
    lib = _lib()
    assert [lib.b2_sample_shard_record_bytes(p) for p in range(-1, 7)] == [0, 8, 3072, 1024, 1024, 1024, 8, 0]
    assert lib.b2_sample_shard_state_bytes() >= 3072


def test_argument_checks_before_any_launch():
    """every bad argument is refused before a launch (no device pointer is ever dereferenced)"""
    lib = _lib()
    p = C.c_void_p(16)  # never dereferenced: the checks come first
    ok = dict(phase=1, rec=p, state=p, all=p, nranks=2, logits=p, rows=4, n=100, ld=100, off=100, n_total=200, ft=9)

    def call(**kw):
        a = {**ok, **kw}
        return lib.b2_sample_shard(a["phase"], a["rec"], a["state"], a["all"], a["nranks"], a["logits"], a["rows"], a["n"],
                                   a["ld"], a["off"], a["n_total"], p, p, p, p, p, a["ft"], None)

    for kw in (dict(phase=-1), dict(phase=6), dict(rec=None), dict(state=None), dict(all=None), dict(logits=None),
               dict(nranks=0), dict(nranks=9), dict(rows=-1), dict(n=0), dict(ld=99), dict(off=-1), dict(off=101),
               dict(n_total=199), dict(ft=7)):
        assert call(**kw) == B2_ERR_PARAM, kw
    assert call(n_total=262145, off=0) == B2_ERR_LIMIT
    assert call(rows=0) == 0  # nothing to launch
    for bad in ((None, p, p, 2, 4), (p, None, p, 2, 4), (p, p, None, 2, 4), (p, p, p, 0, 4), (p, p, p, 9, 4), (p, p, p, 2, -1)):
        assert lib.b2_sample_shard_merge(bad[0], bad[1], bad[2], bad[3], bad[4], p, None) == B2_ERR_PARAM, bad
    assert lib.b2_sample_shard_merge(p, p, p, 2, 4, None, None) == B2_ERR_PARAM


def test_decode_stack_sampling_limits_under_tp():
    """sample=True runs under tensor parallelism; multi-token steps stay refused, and so do sampled verification, fp16
    under tensor parallelism, and a tensor-parallel stack with no way to reach its peers (no process group, no comm)"""
    from b200spark import model
    with pytest.raises(AssertionError, match="q_len == 1"):
        model.DecodeStack(model.TINY, 1, 16, q_len=4, sample=True, device="cpu")
    with pytest.raises(AssertionError, match="single GPU"):
        model.DecodeStack(model.TINY, 1, 16, q_len=4, tp_size=2, sample=True, device="cpu")
    with pytest.raises(AssertionError, match="single GPU"):
        model.DecodeStack(model.TINY, 1, 16, q_len=4, tp_size=2, sampled_verify=True, device="cpu")
    with pytest.raises(AssertionError, match="fp16"):
        model.DecodeStack(model.TINY, 1, 16, tp_size=2, sample=True, dtype=torch.float16, device="cpu")
    with pytest.raises(AssertionError, match="process group"):
        model.DecodeStack(model.TINY, 1, 16, tp_size=2, sample=True, device="cpu")
    with pytest.raises(AssertionError, match="process group"):
        model.DecodeStack(model.TINY, 1, 16, tp_size=2, device="cpu")
