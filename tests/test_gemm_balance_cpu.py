"""CPU: the wgmma GEMM's work schedule (tests/tc_schedule.py, the restatement of make_tc_plan / TcSched): every tile is
walked exactly once, each leftover n-group's head runs first on its CTA and its tail last on another, the k-slices of the
other plans are the k-split plans of gemm_exact, and the kernel's own segment arithmetic (wq_gemm_shared.cuh, compiled for the
host here) walks the same segments."""
import os
import subprocess

import pytest

import gemm_exact as X
import tc_schedule as TS

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# (NG, KT): Qwen2-7B gate+up pair, down, qkv, o, lm_head; a pair with exactly two rounds; Qwen2-72B TP8 shapes; the exact
# tests' shapes (K = 128 and 1000 included); one n-group; one n-group per SM and one more; more than half the SMs left over
SHAPES = [(296, 56), (28, 296), (36, 56), (28, 56), (1188, 56), (264, 56), (10, 128), (64, 16), (58, 58), (11, 2), (4, 16),
          (17, 16), (1, 56), (132, 56), (133, 56), (148, 56), (300, 3), (5, 1), (230, 56)]


def _plans():
    for NG, KT in SHAPES:
        for sms in (132, 114, 7):
            for ms in (1, 2, 6):
                yield TS.plan(NG, KT, sms, ms)
            yield TS.plan(NG, KT, sms, 6, persist=False)


@pytest.mark.parametrize("p", list(_plans()), ids=str)
def test_every_tile_once(p):
    seen = set()
    heads, tails = {}, {}
    for b in range(p.grid):
        segs = p.segments(b)
        assert len(segs) >= 1 and (not p.multi or len(segs) <= p.rounds + 2)
        for i, (ng, kt0, kt1, part, parts, carry) in enumerate(segs):
            assert 0 <= ng < p.NG and 0 <= kt0 < kt1 <= p.KT
            for kt in range(kt0, kt1):
                assert (ng, kt) not in seen, (p, b, ng, kt)
                seen.add((ng, kt))
            if carry == 1:
                assert i == 0 and kt0 == 0
                heads[ng] = (b, kt1)
            if carry == 2:
                assert i == len(segs) - 1 and kt1 == p.KT
                tails[ng] = (b, kt0)
    assert len(seen) == p.NG * p.KT, p
    assert heads.keys() == tails.keys()
    for ng in heads:   # the head ends where the tail starts, on another CTA, a multiple of 4 k-tiles in
        assert heads[ng][1] == tails[ng][1] and heads[ng][0] != tails[ng][0] and heads[ng][1] % 4 == 0


@pytest.mark.parametrize("NG,KT", SHAPES)
@pytest.mark.parametrize("max_split", [1, 6])
def test_plan_matches_the_k_split_plan(NG, KT, max_split):
    """Where no n-group is left over whole-round, the plan is the k-slice plan gemm_exact restates (the same sums)."""
    p = TS.plan(NG, KT, 132, max_split)
    case = X.Case(4, 64 * KT, 128 * NG)
    assert p.multi == (NG > 132) == any(l["multi"] for l in X.launches(case, 64))
    if not p.multi:
        assert p.S == X.tc_split(case, 132, max_split)
    else:
        split = max_split > 1 and 0 < 2 * (NG % 132) <= 132
        assert p.S == 1 and p.h == (KT // 2 // 4 * 4 if split else 0)


def test_benchmark_shapes():
    """The schedules the decode step runs at batch 17-64 (H100, 132 SMs)."""
    lm = TS.plan(1188, 56)
    assert (lm.grid, lm.rounds, lm.h, lm.max_tiles()) == (132, 9, 0, 504)     # lm_head: whole n-groups only
    gu = TS.plan(296, 56)                                                      # gate+up: 2 rounds + a 28-tile half on 64 CTAs
    assert (gu.grid, gu.rounds, gu.h) == (132, 2, 28) and gu.max_tiles() == 140   # not 3 x 56 on 32 CTAs
    for NG, KT, S in ((28, 296, 4), (36, 56, 3), (28, 56, 4)):                 # down, qkv, o: equal k-slices
        p = TS.plan(NG, KT)
        assert (p.grid, p.S) == (NG * S, S)
    one = TS.plan(296, 56, max_split=1)
    assert one.h == 0 and one.max_tiles() == 3 * 56


HARNESS = r"""
#include <cstdio>
#include "wq_gemm_shared.cuh"
int main() {
  int NG, KT, grid, rounds, S, h;
  while (scanf("%d %d %d %d %d %d", &NG, &KT, &grid, &rounds, &S, &h) == 6) {
    for (int b = 0; b < grid; ++b) {
      const b2::TcSched s(NG, KT, grid, rounds, S, h, b);
      for (int i = 0; i < s.count(); ++i) {
        const b2::TcSeg g = s.seg(i);
        printf("%d %d %d %d %d %d ", g.ng, g.kt0, g.kt1, g.part, g.parts, g.carry);
      }
      printf("\n");
    }
  }
  return 0;
}
"""


def test_kernel_segment_arithmetic_matches(tmp_path):
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not os.path.exists(nvcc):
        pytest.skip("no nvcc")
    src, exe = tmp_path / "sched.cu", tmp_path / "sched"
    src.write_text(HARNESS)
    subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-std=c++17", "-I",
                    os.path.join(ROOT, "dash-infer_b200", "csrc"), str(src), "-o", str(exe)], check=True, capture_output=True)
    plans = list(_plans())
    stdin = "".join(f"{p.NG} {p.KT} {p.grid} {p.rounds} {p.S} {p.h}\n" for p in plans)
    lines = iter(subprocess.run([str(exe)], input=stdin, capture_output=True, text=True, check=True).stdout.splitlines())
    for p in plans:
        for b in range(p.grid):
            assert [int(v) for v in next(lines).split()] == [v for seg in p.segments(b) for v in seg], (p, b)
