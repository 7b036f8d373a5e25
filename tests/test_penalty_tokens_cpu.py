"""CPU: the restatement of b2_penalize_tokens (tests/penalty_tokens_ref.py) on hand-worked chains and trees, the restated
bugs it must tell apart, the argument checks of the entry point, and the local memory of the new kernel (cuobjdump), all
without a GPU."""
import ctypes as C
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

import penalty_ref as P
import penalty_tokens_ref as PT

B2_ERR_PARAM, B2_ERR_LIMIT = 3, 4
VOCAB = 48


def _x(rows, ft):
    base = np.array([((i * 7) % 23 - 11) * 0.375 for i in range(VOCAB)], np.float64)
    base[20], base[21] = 0.0, -0.0
    return P.rn(np.stack([base * (1 + 0.3 * (r % 3)) + 0.125 * r for r in range(rows)]), ft)


def _prm(**kw):
    prm = dict(P.neutral(1))
    prm.update(kw)
    return prm


# (name, base history, prompt length, tokens row, parents row or None, params, max_len)
CASES = [
    # a chain with a repeated draft and an out-of-range one; 3 occurs in the prompt and once generated
    ("chain", [3, 5, 3, 9], 2, [9, 7, 3, 7, 60], None,
     _prm(repetition=[1.3], presence=[0.5], frequency=[0.75], no_repeat_ngram=[2], min_length=[7], eos_id=[40],
          suppress=[1]), 64),
    # a tree: node 4's path is 3, 4 (13, 11); its siblings' and cousins' drafts are not its context
    ("tree", [3, 5, 3, 9], 1, [9, 11, 12, 13, 11, 12], [0, 0, 1, 0, 3, 2],
     _prm(repetition=[0.5], presence=[-0.5], frequency=[1.5], no_repeat_ngram=[1], min_length=[6], eos_id=[9],
          suppress=[0]), 64),
    # the slot fills: L = 4, max_len 6, so a path of 3 keeps its first 2 tokens
    ("full", [3, 5, 3, 9], 4, [9, 7, 7, 8], None,
     _prm(repetition=[1.05], frequency=[0.5], no_repeat_ngram=[3], min_length=[7], eos_id=[5]), 6),
    # -1 in the history (an id stored outside the vocabulary): an out-of-range draft compares equal to it
    ("oob", [4, -1, 8, 6], 0, [6, 60, 8, -5], None, _prm(frequency=[0.25], no_repeat_ngram=[2]), 64),
    # the n-gram tail straddles the base / path boundary: 3 9 | 7 matches 3 9 7 ... planted in the base
    ("straddle", [1, 9, 7, 2, 1, 9], 3, [9, 7, 4, 1, 9], None, _prm(no_repeat_ngram=[3], presence=[0.25]), 64),
]


def run(case, ft, bugs=()):
    _, hist, plen, row, par, prm, max_len = case
    T = len(row)
    return PT.penalize_tokens(_x(T, ft), [hist], [plen], [row], None if par is None else [par], prm, ft, max_len, VOCAB,
                              bugs=bugs)


def test_virtual_histories():
    V = lambda hist, plen, row, par, t, ml=64, bugs=(): PT.virtual(hist, plen, row, par, t, ml, VOCAB, bugs)  # noqa: E731
    row = [9, 7, 3, 7, 60]
    assert [V([3, 5, 3, 9], 2, row, None, t)[0] for t in range(5)] == [
        [3, 5, 3, 9], [3, 5, 3, 9, 7], [3, 5, 3, 9, 7, 3], [3, 5, 3, 9, 7, 3, 7], [3, 5, 3, 9, 7, 3, 7, -1]]
    assert V([3, 5, 3, 9], 2, row, None, 4)[1] == 2  # the prompt length stays
    par, row = [0, 0, 1, 0, 3, 2], [9, 11, 12, 13, 11, 12]
    assert PT.path_nodes(par, 4) == [3, 4] and PT.path_nodes(par, 5) == [1, 2, 5] and PT.path_nodes(par, 0) == []
    assert V([1], 0, row, par, 5)[0] == [1, 11, 12, 12]
    assert V([3, 5, 3, 9], 4, [9, 7, 7, 8], None, 3, ml=6)[0] == [3, 5, 3, 9, 7, 7]
    # a parent outside [0, t) is the root
    assert PT.path_nodes([0, 0, 5, -1, 3], 2) == [2] and PT.path_nodes([0, 0, 5, -1, 3], 4) == [3, 4]


@pytest.mark.parametrize("ft", ["bf16", "fp16"])
def test_known_values(ft):
    out, _ = run(CASES[0], ft)
    x = _x(5, ft)
    ban = P.rn(P.BAN, ft)[()]
    R = P.rn(1.3, ft)[()]

    def rep(v):
        return P.rn(v * R if v < 0 else v / R, ft)[()]

    # row 3: V = 3 5 3 9 | 7 3 7: id 7 twice generated, id 5 prompt only (suppress: kept); the 2-gram (7 3) bans 3
    assert out[3, 7] == P.rn(rep(x[3, 7]) - P.rn(2 * 0.75 + 0.5, ft), ft)[()]
    assert out[3, 5] == x[3, 5] and out[3, 3] == ban
    # row 2: V = 3 5 3 9 | 7 3: id 3 twice generated (once in the base, once on the path)
    assert out[2, 3] == P.rn(rep(x[2, 3]) - P.rn(2 * 0.75 + 0.5, ft), ft)[()]
    assert out[0, 7] == x[0, 7]  # not in row 0's context
    assert out[1, 7] == P.rn(rep(x[1, 7]) - P.rn(0.75 + 0.5, ft), ft)[()]
    # 2-gram: row 2 ends in 3, which was followed by 5 and by 9; row 1 ends in 7, which occurs nowhere before
    assert out[2, 5] == out[2, 9] == ban and out[1, 5] != ban
    # min_length 7 against L' = 4, 5, 6, 7, 8
    assert [out[t, 40] == ban for t in range(5)] == [True, True, True, False, False]
    # the tree: node 4's context is 13 11 (one 11), node 5's is 11 12 12; g == 1 bans every id of V
    out, _ = run(CASES[1], ft)
    assert out[4, 11] == out[4, 13] == out[4, 3] == ban and out[4, 12] != ban
    assert out[5, 12] == out[5, 11] == ban and out[5, 13] != ban
    assert out[0, 9] == ban and out[1, 9] == ban  # eos: L' = 4, 5 < 6


def test_straddling_ngram():
    out, _ = run(CASES[4], "bf16")
    ban = P.rn(P.BAN, "bf16")[()]
    # row 1: V = 1 9 7 2 1 9 | 7, tail (9 7) -> 2 banned; row 2: ... 9 7 4, tail (7 4) -> nothing; row 4: ... 1 9 -> 7
    assert out[1, 2] == ban and not (out[2] == ban).any() and out[4, 7] == ban and out[0, 7] == ban


@pytest.mark.parametrize("ft", ["bf16", "fp16"])
def test_q_len_one_is_penalize(ft):
    for case in CASES:
        _, hist, plen, row, par, prm, max_len = case
        x = _x(1, ft)
        got, _ = PT.penalize_tokens(x, [hist], [plen], [row[:1]], None, prm, ft, max_len, VOCAB)
        tok = np.array([hist], np.int64)
        want, _ = P.penalize(x, tok, [len(hist)], [plen], prm, ft)
        assert np.all(P.same(got, want))


@pytest.mark.parametrize("bug", PT.BUGS)
def test_each_bug_changes_an_output(bug):
    changed = 0
    for case in CASES:
        for ft in ("bf16", "fp16"):
            out, alt = run(case, ft)
            bad, _ = run(case, ft, bugs=(bug,))
            changed += int(np.sum(~(P.same(bad, out) | P.same(bad, alt))))
    assert changed > 0, bug


def test_argument_checks_without_gpu():
    """every bad argument returns its status before any launch (fake, never dereferenced pointers)"""
    from b200spark import _lib
    lib = _lib.lib
    p = 0x1000
    h = _lib.TokenHistory(p, p, p, p, p, p, 16, 100)
    prm = _lib.PenaltyParams(p, p, p, p, p, p, p, None)
    ok = dict(logits=p, batch=2, q_len=4, parents=p, tokens=p, n=100, ld=100, off=0, h=h, prm=prm, ft=_lib.DT_BF16)
    call = lambda a: lib.b2_penalize_tokens(a["logits"], a["batch"], a["q_len"], a["parents"], a["tokens"], a["n"],  # noqa
                                            a["ld"], a["off"], C.byref(a["h"]), C.byref(a["prm"]), a["ft"], None)
    for bad, want in ((dict(logits=None), B2_ERR_PARAM), (dict(tokens=None), B2_ERR_PARAM), (dict(batch=-1), B2_ERR_PARAM),
                      (dict(n=0), B2_ERR_PARAM), (dict(ld=99), B2_ERR_PARAM), (dict(off=-1), B2_ERR_PARAM),
                      (dict(off=1), B2_ERR_PARAM), (dict(ft=_lib.DT_F32), B2_ERR_PARAM),
                      (dict(h=_lib.TokenHistory(p, p, p, None, p, p, 16, 100)), B2_ERR_PARAM),
                      (dict(h=_lib.TokenHistory(p, p, p, p, p, p, 0, 100)), B2_ERR_PARAM),
                      (dict(prm=_lib.PenaltyParams(p, p, p, p, p, None, p, None)), B2_ERR_PARAM),
                      (dict(q_len=0), B2_ERR_LIMIT), (dict(q_len=17), B2_ERR_LIMIT), (dict(batch=1 << 29), B2_ERR_LIMIT),
                      (dict(q_len=0, batch=-1), B2_ERR_PARAM)):
        assert call(dict(ok, **bad)) == want, bad
    assert call(dict(ok, batch=0)) == 0  # nothing to do, nothing launched
    assert call(dict(ok, batch=0, parents=None)) == 0


def test_front_end_checks():
    import torch
    from b200spark import ops
    h, pen = ops.TokenHistory(2, 8, 50, device="cpu"), ops.Penalties(2, device="cpu")
    tk = torch.zeros(2, 4, dtype=torch.int64)
    for lg, t, par in ((torch.zeros(7, 50, dtype=torch.bfloat16), tk, None),
                       (torch.zeros(8, 50, dtype=torch.bfloat16), tk.int(), None),
                       (torch.zeros(8, 50, dtype=torch.bfloat16), tk, torch.zeros(2, 4, dtype=torch.int64)),
                       (torch.zeros(12, 50, dtype=torch.bfloat16), torch.zeros(3, 4, dtype=torch.int64), None)):
        with pytest.raises(AssertionError, match="penalize_tokens|"):
            ops.penalize_tokens(lg, h, pen, t, par)


ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "dash-infer_b200", "lib", "libb200spark.so")
CUOBJDUMP = shutil.which("cuobjdump") or next((p for p in ("/usr/local/cuda/bin/cuobjdump",) if os.path.exists(p)), None)


@pytest.mark.skipif(CUOBJDUMP is None, reason="cuobjdump not found")
def test_kernel_has_no_local_memory():
    out = subprocess.run([CUOBJDUMP, "-res-usage", LIB], check=True, capture_output=True, text=True).stdout
    usage, cur = {}, None
    for line in out.splitlines():
        m = re.match(r"\s*Function (\S+):", line)
        if m:
            cur = m.group(1)
        elif cur is not None and "REG:" in line:
            usage[cur] = (int(re.search(r"STACK:(\d+)", line).group(1)), int(re.search(r"LOCAL:(\d+)", line).group(1)))
            cur = None
    new = {k: v for k, v in usage.items() if "penalize_tokens_kernel" in k}
    assert len(new) == 2, sorted(new)
    assert all(v == (0, 0) for v in new.values()), new
