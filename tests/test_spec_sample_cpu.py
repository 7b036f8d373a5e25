"""CPU: sampled speculative verification (tests/spec_sample_ref.py), the entry points' argument checks and the
DecodeStack refusals, without a GPU.

Over the context-hash oracle, single-token sampling and the speculative loop emit the same tokens and end at the same
offsets for every tree family, T from 2 to 16, four drafters and mixed per-sequence parameters (greedy included); each
restated bug of MUTATIONS breaks that equality or the step's outputs; bad arguments return B2_ERR_PARAM / B2_ERR_LIMIT
before any launch; the new kernels have no stack frame."""
import ctypes as C
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

import spec_sample_ref as SS

B2_ERR_PARAM, B2_ERR_LIMIT = 3, 4
VOCAB = 512
OFFSETS = np.array([0, 2 ** 32 - 3, 17, 2 ** 63 + 5], np.uint64)


def _prompts(B):
    return [[b + 1, 7 * b + 3, 11] for b in range(B)]


def _references(oracle, params, L):
    B = len(OFFSETS)
    return [SS.sample_stream(oracle, _prompts(B)[b], params, b, OFFSETS[b], L)[0] for b in range(B)]


def _run(tree, T, drafter, L=16, variant=None, seed=0):
    """(streams equal and offsets equal?, accepted counts per step) of one speculative run against single-token sampling"""
    oracle = SS.Oracle(VOCAB, seed=seed)
    params = SS.params_of(len(OFFSETS), seed)
    truths = _references(oracle, params, L + 16)
    out, off, counts = SS.spec_stream(oracle, _prompts(len(OFFSETS)), params, OFFSETS, L, T, tree, drafter, seed=seed,
                                      truths=truths, variant=variant)
    ref = _references(oracle, params, max(len(o) for o in out))
    ok = all(out[b] == ref[b][:len(out[b])] for b in range(len(out)))
    ok = ok and all(off[b] == OFFSETS[b] + np.uint64(len(out[b])) for b in range(len(out)))
    return ok, counts


@pytest.mark.parametrize("drafter", SS.DRAFTERS)
@pytest.mark.parametrize("T", [2, 3, 5, 8, 16])
@pytest.mark.parametrize("tree", list(SS.TREES))
def test_stream_equality(tree, T, drafter):
    """the speculative loop emits exactly single-token sampling's tokens and leaves the offsets where it leaves them"""
    ok, counts = _run(tree, T, drafter)
    assert ok
    if drafter in ("truth", "argmax"):  # drafts that know the likely continuation are accepted: the test is not vacuous
        assert max(int(c.max()) for c in counts) > 1


def _walk_case():
    """node 1 and 2 are children of the root with the same draft, node 3 continues node 1: the lowest-index child gives
    the path [0, 1, 3]; node 4 hangs below 3 with a draft that equals its own draw but not 3's"""
    tokens = np.array([[5, 9, 9, 4, 6]])
    pred = np.array([[9, 4, 8, 7, 6]])
    return tokens, pred, np.array([[0, 0, 0, 1, 3]], np.int32)


def test_walk_and_advance():
    tokens, pred, par = _walk_case()
    n, paths, nxt = SS.accept(tokens, pred, par)
    assert list(n) == [3] and paths == [[0, 1, 3]] and list(nxt) == [7]
    assert SS.advance(np.array([10], np.uint64), n, 5)[0] == 13
    n, paths, nxt = SS.accept(tokens, pred)  # a chain: 9 == pred[0], then 9 != pred[1]
    assert list(n) == [2] and list(nxt) == [4]
    # the counters of a tree are offsets + depth, of a chain offsets + t
    ctr = SS.counters(np.array([100], np.uint64), par, 1, 5)
    assert list(ctr[0]) == [100, 101, 101, 102, 103]
    assert list(SS.counters(np.array([100], np.uint64), None, 1, 5)[0]) == [100, 101, 102, 103, 104]


@pytest.mark.parametrize("variant", SS.MUTATIONS)
def test_mutations_break_equality_or_the_step(variant):
    """every restated bug breaks stream equality on one of a few runs, or changes the constructed walk's outputs"""
    tokens, pred, par = _walk_case()
    walk = [SS.accept(tokens, pred, par, variant), SS.advance(np.array([10], np.uint64), SS.accept(tokens, pred, par)[0], 5,
                                                               variant)]
    good = [SS.accept(tokens, pred, par), SS.advance(np.array([10], np.uint64), SS.accept(tokens, pred, par)[0], 5)]
    walk_broken = not (np.array_equal(walk[0][0], good[0][0]) and walk[0][1] == good[0][1] and np.array_equal(walk[1], good[1]))
    stream_broken = any(not _run(tree, T, "truth", L=8, variant=variant)[0]
                        for tree, T in (("chain", 4), ("star", 4), ("topk", 8)))
    assert walk_broken or stream_broken, variant


def test_argument_checks_without_gpu():
    """every rejected call returns before a launch (the addresses are never dereferenced)"""
    from b200spark import _lib
    lib, bf = _lib.lib, _lib.DT_BF16
    A = 1 << 20
    # b2_sample_tokens(ids, logits, batch, q_len, parents, n, ld, t, k, p, seeds, offsets, ft, stream)
    ok = [A, A, 2, 4, None, 100, 100, A, A, A, A, A, bf]
    for i in (0, 1, 7, 8, 9, 10, 11):  # each required pointer NULL
        a = list(ok)
        a[i] = None
        assert lib.b2_sample_tokens(*a, None) == B2_ERR_PARAM, i
    for i, v in ((2, -1), (5, 0), (6, 99), (12, _lib.DT_F32), (12, _lib.DT_I8)):
        a = list(ok)
        a[i] = v
        assert lib.b2_sample_tokens(*a, None) == B2_ERR_PARAM, (i, v)
    for i, v in ((3, 0), (3, 17), (5, _lib.SAMPLE_MAX_N + 1)):
        a = list(ok)
        a[i] = v
        a[6] = max(a[5], a[6])
        assert lib.b2_sample_tokens(*a, None) == B2_ERR_LIMIT, (i, v)
    a = list(ok)
    a[2] = 0
    assert lib.b2_sample_tokens(*a, None) == 0  # no sequences: nothing to launch
    a[4] = A
    assert lib.b2_sample_tokens(*a, None) == 0
    # b2_spec_accept_sampled(accepted, path, next_ids, old, new, tokens, pred, parents, offsets, batch, q_len, stream)
    one = C.c_void_p(16)
    ok = [one, None, None, one, one, one, one, None, one, 2, 4]
    for i in (0, 3, 4, 5, 6, 8):
        a = list(ok)
        a[i] = None
        assert lib.b2_spec_accept_sampled(*a, None) == B2_ERR_PARAM, i
    for path, par in ((one, None), (None, one)):  # path NULL iff parents NULL
        a = list(ok)
        a[1], a[7] = path, par
        assert lib.b2_spec_accept_sampled(*a, None) == B2_ERR_PARAM
    a = list(ok)
    a[9] = -1
    assert lib.b2_spec_accept_sampled(*a, None) == B2_ERR_PARAM
    for T in (0, 17):
        a = list(ok)
        a[10] = T
        assert lib.b2_spec_accept_sampled(*a, None) == B2_ERR_LIMIT
    a = list(ok)
    a[9] = 0
    assert lib.b2_spec_accept_sampled(*a, None) == 0


def test_decode_stack_refusals():
    from b200spark import model
    for kw, msg in ((dict(q_len=4, penalties=True), "penalties"), (dict(q_len=4, tp_size=2), "single GPU"),
                    (dict(q_len=1), "q_len > 1"), (dict(q_len=4, sample=True), "q_len == 1"),
                    (dict(q_len=4, tree=True, penalties=True), "penalties")):
        with pytest.raises(AssertionError, match=msg):
            model.DecodeStack(model.TINY, 1, 16, sampled_verify=True, device="cpu", **kw)


ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "dash-infer_b200", "lib", "libb200spark.so")
CUOBJDUMP = shutil.which("cuobjdump") or next((p for p in ("/usr/local/cuda/bin/cuobjdump",) if os.path.exists(p)), None)


@pytest.mark.skipif(CUOBJDUMP is None, reason="cuobjdump not found")
def test_kernels_have_no_local_memory():
    """no stack frame in the step form of the sampler or in the sampled accept"""
    out = subprocess.run([CUOBJDUMP, "-res-usage", LIB], check=True, capture_output=True, text=True).stdout
    usage, cur = {}, None
    for line in out.splitlines():
        m = re.match(r"\s*Function (\S+):", line)
        if m:
            cur = m.group(1)
        elif cur is not None and "REG:" in line:
            usage[cur] = int(re.search(r"STACK:(\d+)", line).group(1))
            cur = None
    new = {k: v for k, v in usage.items() if "sample_tokens_kernel" in k or "spec_accept_sampled_kernel" in k}
    assert len(new) == 4, sorted(new)
    assert all(v == 0 for v in new.values()), new
