"""CPU: the restatement of b2_ngram_draft and b2_history_append_tokens (tests/ngram_ref.py) on hand-worked cases, the
restated bugs it must tell apart, the argument checks of both entry points, the DecodeStack refusals of `ngram`, and the
local memory of the new kernels (cuobjdump), all without a GPU."""
import ctypes as C
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

import ngram_ref as N
import penalty_ref as P

B2_ERR_PARAM, B2_ERR_LIMIT = 3, 4


def test_period_three_loop():
    S = [5, 1, 2, 3, 1, 2, 3, 1, 2, 3]
    assert [N.match_len(S, e, 4) for e in range(9)] == [0, 0, 0, 3, 0, 0, 4, 0, 0]
    assert N.candidates(S, 1, 4, 2) == [6]  # only the longest match
    assert N.candidates(S, 1, 2, 2) == [6, 3]
    assert N.draft(S, 3, 9, 1, 4, 1, False) == ([3, 1, 2, 3, 1, 2, 3, 1, 2], None, 8)  # the loop goes on past the history
    # periods 3 and 6 continue identically: the trie merges them into one chain
    assert N.draft(S, 3, 6, 1, 2, 2, True) == ([3, 1, 2, 3, 1, 2], [0, 0, 1, 2, 3, 4], 5)


def test_earliest_possible_match():
    """the only match ends at e = n* - 1: its n-gram starts at position 0"""
    S = [7, 8, 9, 1, 2, 3, 4, 7, 8, 9]
    assert N.candidates(S, 3, 4, 1) == [2]
    assert N.draft(S, 9, 5, 3, 4, 1, False) == ([9, 1, 2, 3, 4], None, 4)


def test_no_match():
    for S, n_min in (([1, 2, 3, 4], 1), ([1, 2, 5, 3, 2], 2), ([4], 1), ([], 1)):
        assert N.draft(S, 9, 4, n_min, 4, 1, False) == ([9, 9, 9, 9], None, 0), S
        assert N.draft(S, 9, 4, n_min, 4, 3, True) == ([9, 9, 9, 9], [0, 0, 0, 0], 0), S


def test_n_min_equal_n_max():
    S = [1, 2, 9, 2, 5, 1, 2]
    assert N.candidates(S, 2, 2, 1) == [1]   # only the bigram (1, 2) at e = 1
    assert N.candidates(S, 1, 1, 1) == [3]   # unigrams: the most recent 2
    assert N.draft(S, 2, 4, 2, 2, 1, False)[0] == [2, 9, 2, 5]
    assert N.draft(S, 2, 4, 1, 1, 1, False)[0] == [2, 5, 1, 2]


def test_equal_continuations_tie():
    """three candidates: the most recent and the oldest continue alike and merge; the middle one branches"""
    S = [9, 1, 2, 9, 1, 3, 9, 1, 2, 9]
    assert N.candidates(S, 1, 1, 3) == [6, 3, 0]
    toks, pars, nd = N.draft(S, 9, 6, 1, 1, 3, True)
    # level 1: 1 (all three); level 2: 2 (ranks 0, 2), 3 (rank 1); level 3: 9, 9; level 4: 1 below the first 9
    assert (toks, pars, nd) == ([9, 1, 2, 3, 9, 9], [0, 0, 1, 1, 2, 3], 5)


def test_breadth_first_differs_from_depth_first():
    S = [9, 6, 7, 8, 9, 1, 4, 5, 9, 1, 2, 3, 9]
    assert N.candidates(S, 1, 1, 3) == [8, 4, 0]
    toks, pars, _ = N.draft(S, 9, 8, 1, 1, 3, True)
    assert toks == [9, 1, 6, 2, 4, 7, 3, 5] and pars == [0, 0, 0, 1, 1, 2, 3, 4]
    dtoks, dpars, _ = N.draft(S, 9, 8, 1, 1, 3, True, bugs=("depth_first",))
    assert dtoks == [9, 1, 2, 3, 9, 1, 2, 3] and dpars == [0, 0, 1, 2, 3, 4, 5, 6]  # the first candidate's path only


def test_minus_one_entries():
    """-1 compares like any id; a draft that would be -1 is written as tokens[b][0]"""
    S = [-1, 4, -1, 7, -1, 4, -1]
    assert [N.match_len(S, e, 4) for e in range(6)] == [1, 0, 3, 0, 1, 0]  # e = 2: -1 4 -1
    assert N.draft(S, 8, 5, 1, 4, 1, False) == ([8, 7, 8, 4, 8], None, 4)
    assert N.candidates(S, 1, 1, 2) == [4, 2]
    assert N.draft(S, 8, 5, 1, 1, 2, True) == ([8, 4, 7, 8, 8], [0, 0, 0, 1, 2], 4)


def _bug_cases():
    """hand-worked histories plus random ones over a small vocabulary (many matches, branching tries)"""
    cases = [([5, 1, 2, 3, 1, 2, 3, 1, 2, 3], 6, 1, 4), ([7, 8, 9, 1, 2, 3, 4, 7, 8, 9], 5, 3, 4),
             ([1, 2, 9, 2, 5, 1, 2], 4, 1, 4), ([9, 1, 2, 9, 1, 3, 9, 1, 2, 9], 6, 1, 1),
             ([9, 6, 7, 8, 9, 1, 4, 5, 9, 1, 2, 3, 9], 8, 1, 1), ([1, 2, 3, 4], 4, 1, 4)]
    rng = np.random.default_rng(3)
    for _ in range(40):
        L = int(rng.integers(2, 40))
        cases.append((rng.integers(0, 4, L).tolist(), int(rng.integers(2, 17)), int(rng.integers(1, 3)), 4))
    return cases


DRAFT_BUGS = [b for b in N.BUGS if not b.startswith("append")]
APPEND_BUGS = [b for b in N.BUGS if b.startswith("append")]


@pytest.mark.parametrize("bug", DRAFT_BUGS)
def test_each_drafter_bug_changes_an_output(bug):
    changed = 0
    for S, T, n_min, n_max in _bug_cases():
        for width, tree in ((1, False), (1, True), (min(3, T - 1), True), (T - 1, True)):
            changed += N.draft(S, 0, T, n_min, n_max, width, tree) != N.draft(S, 0, T, n_min, n_max, width, tree, (bug,))
    assert changed > 0, bug


def _append_case():
    pred = [[10, 11, 12, 13], [20, 21, 22, 23], [30, 31, 32, 33]]
    return pred, [3, 1, 4], [[0, 2, 3, 0], [0, 0, 0, 0], [0, 1, 2, 3]]


@pytest.mark.parametrize("bug", APPEND_BUGS)
def test_each_append_bug_changes_an_output(bug):
    pred, acc, path = _append_case()
    good, bad = P.History(3, 16, 100), P.History(3, 16, 100)
    for h in (good, bad):
        h.load(0, [1, 10]); h.load(1, [2, 20]); h.load(2, [3, 30])
    N.append_tokens(good, pred, acc, path)
    N.append_tokens(bad, pred, acc, path, (bug,))
    assert good.tokens != bad.tokens


def test_append_equals_successive_single_appends():
    pred, acc, path = _append_case()
    h = P.History(3, 6, 100)
    h.load(0, [1, 10], 2); h.load(1, [2, 20], 2); h.load(2, [3, 4, 30], 3)
    N.append_tokens(h, pred, acc, path)
    assert N.emitted(pred, acc, path) == [[10, 12, 13], [20], [30, 31, 32, 33]]
    assert h.tokens == [[1, 10, 10, 12, 13], [2, 20, 20], [3, 4, 30, 30, 31, 32]]  # slot 2 stops at max_len 6
    assert h.table(0) == {1: P.IN_PROMPT, 10: P.IN_PROMPT | 1, 12: 1, 13: 1}


def test_argument_checks_without_gpu():
    """every bad argument returns its status before any launch (fake, never dereferenced pointers)"""
    from b200spark import _lib
    lib = _lib.lib
    p = 0x1000
    h = _lib.TokenHistory(p, p, p, p, p, p, 64, 100)
    ok = dict(tokens=p, parents=p, n_draft=p, h=h, batch=2, q_len=8, n_min=1, n_max=4, width=3)
    call = lambda a: lib.b2_ngram_draft(a["tokens"], a["parents"], a["n_draft"], C.byref(a["h"]), a["batch"], a["q_len"],  # noqa
                                        a["n_min"], a["n_max"], a["width"], None)
    for bad, want in ((dict(tokens=None), B2_ERR_PARAM), (dict(h=_lib.TokenHistory(None, p, p, p, p, p, 64, 100)), B2_ERR_PARAM),
                      (dict(h=_lib.TokenHistory(p, None, p, p, p, p, 64, 100)), B2_ERR_PARAM),
                      (dict(h=_lib.TokenHistory(p, p, p, p, p, p, 0, 100)), B2_ERR_PARAM),
                      (dict(batch=-1), B2_ERR_PARAM), (dict(n_min=0), B2_ERR_PARAM), (dict(n_min=5), B2_ERR_PARAM),
                      (dict(width=0), B2_ERR_PARAM), (dict(width=8), B2_ERR_PARAM), (dict(parents=None), B2_ERR_PARAM),
                      (dict(q_len=1, width=1), B2_ERR_LIMIT), (dict(q_len=17), B2_ERR_LIMIT), (dict(n_max=17), B2_ERR_LIMIT)):
        assert call(dict(ok, **bad)) == want, bad
    assert call(dict(ok, batch=0)) == 0  # nothing to do, nothing launched
    assert call(dict(ok, batch=0, parents=None, width=1, n_draft=None)) == 0
    app = lambda hh=h, pred=p, acc=p, path=p, batch=2, q_len=4: lib.b2_history_append_tokens(  # noqa
        C.byref(hh), pred, acc, path, batch, q_len, None)
    for bad, want in ((dict(pred=None), B2_ERR_PARAM), (dict(acc=None), B2_ERR_PARAM), (dict(batch=-1), B2_ERR_PARAM),
                      (dict(hh=_lib.TokenHistory(p, p, p, None, p, p, 64, 100)), B2_ERR_PARAM),
                      (dict(hh=_lib.TokenHistory(p, p, p, p, p, p, 1 << 30, 100)), B2_ERR_PARAM),
                      (dict(q_len=0), B2_ERR_LIMIT), (dict(q_len=17), B2_ERR_LIMIT)):
        assert app(**bad) == want, bad
    assert app(batch=0) == 0 and app(batch=0, path=None) == 0


def test_stack_refusals():
    from b200spark import model
    for kw in (dict(q_len=1, ngram=(1, 4, 1)), dict(q_len=4, ngram=(1, 4, 2)), dict(q_len=4, ngram=(0, 4, 1)),
               dict(q_len=4, ngram=(3, 2, 1)), dict(q_len=4, ngram=(1, 17, 1)), dict(q_len=4, tree=True, ngram=(1, 4, 4)),
               dict(q_len=4, tree=True, ngram=(1, 4, 0))):
        with pytest.raises(AssertionError, match="ngram"):
            model.DecodeStack(model.TINY, 1, 16, device="cpu", **kw)
    with pytest.raises(AssertionError, match="penalties"):  # penalties stay single-token with a drafter too
        model.DecodeStack(model.TINY, 1, 16, device="cpu", q_len=4, penalties=True, ngram=(1, 4, 1))


ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "dash-infer_b200", "lib", "libb200spark.so")
CUOBJDUMP = shutil.which("cuobjdump") or next((p for p in ("/usr/local/cuda/bin/cuobjdump",) if os.path.exists(p)), None)


@pytest.mark.skipif(CUOBJDUMP is None, reason="cuobjdump not found")
def test_kernels_have_no_local_memory():
    out = subprocess.run([CUOBJDUMP, "-res-usage", LIB], check=True, capture_output=True, text=True).stdout
    usage, cur = {}, None
    for line in out.splitlines():
        m = re.match(r"\s*Function (\S+):", line)
        if m:
            cur = m.group(1)
        elif cur is not None and "REG:" in line:
            usage[cur] = (int(re.search(r"STACK:(\d+)", line).group(1)), int(re.search(r"LOCAL:(\d+)", line).group(1)))
            cur = None
    new = {k: v for k, v in usage.items() if "ngram_draft_kernel" in k or "history_append_tokens_kernel" in k}
    assert len(new) == 2, sorted(new)
    assert all(v == (0, 0) for v in new.values()), new
