"""CPU: the cluster form of the wgmma GEMM's k-sliced plans (make_tc_plan in wq_gemm.cu, over the schedule tests/tc_schedule.py
restates).  A plan of k-slices (rounds == 0, S > 1) runs its S slices of an n-group as one cluster of S consecutive CTAs when
clusters are on (B2_GEMM_TC_CLUSTER), S is at most the portable cluster size 8 and the occupancy query says all NG clusters are
resident at once; else it keeps the workspace split.  A cluster is then exactly the slices of one n-group, in k order on
ranks 0..S-1, the cluster size divides the grid, every tile is still walked once, and the slices finish disjoint shares of
the tile's rows that together cover them all."""
import pytest

import tc_schedule as TS
from test_gemm_balance_cpu import SHAPES

MAX_CLUSTER = 8  # kTcMaxCluster


def cluster_size(p, fits=True):
    """CTAs per cluster make_tc_plan picks for plan p; fits: clusters are on and the occupancy query accepts NG of them."""
    return p.S if p.rounds == 0 and 1 < p.S <= MAX_CLUSTER and fits else 1


def _plans():
    for NG, KT in SHAPES:
        for sms in (132, 114, 7):
            for ms in (1, 2, 3, 4, 6, 8, 12):
                for fits in (True, False):
                    yield TS.plan(NG, KT, sms, ms), fits


@pytest.mark.parametrize("p,fits", list(_plans()), ids=str)
def test_clusters_are_the_slices_of_one_n_group(p, fits):
    c = cluster_size(p, fits)
    assert p.grid % c == 0
    seen = set()
    for c0 in range(0, p.grid, c):
        segs = [s for b in range(c0, c0 + c) for s in p.segments(b)]
        if c > 1:
            assert len(segs) == c                                              # one k-slice per CTA
            assert {s[0] for s in segs} == {c0 // c}                           # one n-group per cluster
            assert [s[3] for s in segs] == list(range(c))                      # slice r on cluster rank r
            assert [s[1] for s in segs[1:]] == [s[2] for s in segs[:-1]]       # in k order
            assert segs[0][1] == 0 and segs[-1][2] == p.KT
        for ng, kt0, kt1, *_ in segs:
            for kt in range(kt0, kt1):
                assert (ng, kt) not in seen
                seen.add((ng, kt))
    assert len(seen) == p.NG * p.KT


@pytest.mark.parametrize("S", range(2, MAX_CLUSTER + 1))
@pytest.mark.parametrize("M", [1, 5, 16, 17, 33, 64])
def test_cluster_rows_partition_the_tile(S, M):
    """Rank r finishes rows r, r + S, ... (wq_gemm_tc.cu: rows = (M - r + S - 1) / S of them)."""
    rows = [[(u * S + r) for u in range((M - r + S - 1) // S)] for r in range(S)]
    assert sorted(m for rr in rows for m in rr) == list(range(M))


def test_benchmark_shapes_run_as_clusters():
    """down, qkv and o at batch 17-64 on an H100: clusters of 4, 3 and 4 k-slices; gate+up and lm_head (more n-groups
    than SMs) keep their persistent schedule."""
    for NG, KT, S in ((28, 296, 4), (36, 56, 3), (28, 56, 4)):
        p = TS.plan(NG, KT)
        assert (p.grid, p.S, cluster_size(p)) == (NG * S, S, S)
        assert cluster_size(p, fits=False) == 1
    assert cluster_size(TS.plan(296, 56)) == 1 and cluster_size(TS.plan(1188, 56)) == 1
