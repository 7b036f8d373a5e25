"""CPU: the SpanAttention work-split mirror and the needle inputs of tests/test_attn_needles_gpu.py.

  * the mirror's invariants (pieces tile each (sequence, kv-head), at most two partial slots per CTA, slot parity only on a
    first piece, no level-1 slot shared by two (sequence, kv-head)s, merge fan-in within kMergeMaxSrc) for random batches
    and grids and for every launch the GPU file makes;
  * every merge shape the GPU file needs occurs;
  * teeth: on the CPU quantizers' cache of every GPU case, removing any needle or moving it by one token moves its head's
    fp64 output by >= 20 envelopes, while the kernel's own rounding (simulated) stays inside one.
The default-knob grid is the SM count times the CTAs per SM; here 132 SMs (H100 SXM) and 1 or 2 CTAs per SM stand in."""
import numpy as np
import pytest

import attn_needles as A

H100_SMS = 132
DEFAULT_GRIDS = (H100_SMS, 2 * H100_SMS)


def test_mirror_invariants_random_batches():
    rng = np.random.default_rng(0)
    seen = set()
    for _ in range(3000):
        B = int(rng.integers(1, 9))
        lens = [int(x) for x in rng.integers(1, 9000, B)]
        if rng.random() < 0.3:
            lens = [int(x) for x in rng.integers(1, 200, B)]
        nG = int(rng.choice([1, 2, 4, 8]))
        grid = int(rng.choice([8, 33, 114, 132, 264, 396, 528]))
        mp = int(rng.integers(1, 40)) if rng.random() < 0.3 else None
        dec = A.decompose(lens, nG, grid, mp)
        A.check_decomposition(dec, lens)
        seen |= {bg.merge for bg in dec.bgs}
    assert seen == {"single", "direct", "two-level"}


def test_mirror_matches_hand_worked_split():
    """Two sequences of 130 and 64 tokens, 2 kv-heads, 4 CTAs: 8 tiles, Tc = 2."""
    dec = A.decompose([130, 64], 2, 4)
    assert dec.Tc == 2 and dec.total == 8
    first = dec.bgs[0]  # (b 0, g 0): tiles 0..2 -> CTA 0 (tiles 0, 1) and CTA 1 (tile 2)
    assert [(p.cta, p.tok_lo, p.tok_hi) for p in first.pieces] == [(0, 0, 128), (1, 128, 130)]
    second = dec.bgs[1]  # (b 0, g 1): tiles 3..5 -> starts inside CTA 1: slot parity 1
    assert second.first_par == 1 and [p.slot_written for p in second.pieces] == [3, 4]
    assert [bg.npieces for bg in dec.bgs] == [2, 2, 1, 1]


@pytest.mark.parametrize("grid", [114, H100_SMS, 144])
def test_merge_shapes_found(grid):
    found = set()
    for lens, nH, nG, mp in A.merge_shape_cases(grid):
        dec = A.decompose(lens, nG, grid, mp)
        A.check_decomposition(dec, lens)
        found |= A.shapes(dec)
    assert found == A.MERGE_SHAPES, A.MERGE_SHAPES - found


def test_mirror_invariants_of_every_gpu_launch():
    for case in A.tile_cases() + A.long_cases() + A.stale_cases():
        for grid in DEFAULT_GRIDS:
            A.check_decomposition(A.decompose(case.lens, case.nG, grid, case.max_pieces), case.lens)
    for case in A.merge_cases(H100_SMS):
        A.check_decomposition(A.decompose(case.lens, case.nG, H100_SMS, case.max_pieces), case.lens)


def _teeth(case, grid):
    prob = case.problem()
    worst_teeth, worst_honest = np.inf, 0.0
    for needles, stale in case.rounds(grid):
        k_rows, v_rows, q = prob.rows(needles)
        kc, ks, vc, vs = A.cpu_caches(k_rows, v_rows, case.mode)
        res = A.evaluate(prob, q, kc, ks, vc, vs, case.mode, needles, stale=stale)
        assert res.honest <= 1.0, (case.name, res.honest)
        if max(case.lens) > 1:
            assert res.teeth >= A.TEETH, (case.name, res.teeth, res.weakest)
        worst_teeth, worst_honest = min(worst_teeth, res.teeth), max(worst_honest, res.honest)
    print("%s: least teeth %.1f envelopes, simulated rounding %.2f of the envelope" % (case.name, worst_teeth, worst_honest))


@pytest.mark.parametrize("case", A.tile_cases(), ids=lambda c: c.name)
def test_teeth_tile_edges(case):
    _teeth(case, H100_SMS)


@pytest.mark.parametrize("case", [c for m in (A.NONE, A.I8, A.FP8) for c in A.merge_cases(H100_SMS, m)] + A.stale_cases() +
                         A.head64_cases(), ids=lambda c: c.name)
def test_teeth_merge_stale_head64(case):
    _teeth(case, H100_SMS)


@pytest.mark.parametrize("case", A.long_cases(), ids=lambda c: c.name)
def test_teeth_ctx_32768(case):
    _teeth(case, 2 * H100_SMS)


def test_needles_dominate_and_rounding_is_sized():
    """A lone needle at L = 4100 carries most of its head's weight; bf16 P rounding alone is above 2e-3 in a cancelling
    element, which is why the envelope has a probability term."""
    case = A.Case("one", A.NONE, A.BF16, 128, 8, 1, [4100])
    prob = case.problem()
    needles = [(0, 0, 1234, 0.0)]
    k_rows, v_rows, q = prob.rows(needles)
    kc, ks, vc, vs = A.cpu_caches(k_rows, v_rows, A.NONE)
    K = kc[0][0] * ks[0][0][:, None]
    s = K @ q[0, 0].astype(np.float64) / np.sqrt(128)
    p = np.exp(s - s.max())
    p /= p.sum()
    assert p[1234] > 0.85
    u_p, _ = A.p_type(A.NONE, A.BF16, 128)
    assert u_p * p[1234] * np.abs(vc[0][0, 1234]).max() > 2e-3 / 2
