"""CPU: tree-structured verification's restatements (tests/tree_ref.py) — chains reduce to the multi-token step, the tree
accept rule on hand-written trees, compaction and its read-before-write hazard — and the argument checks of the tree
entry points that fail before touching the device."""
import ctypes as C

import numpy as np
import pytest

import spec_ref as S
import tree_ref as TR
from oracle import kvcache_ref as KV


def test_depth_anc():
    assert TR.depth_anc(TR.chain(5)) == ([0, 1, 2, 3, 4], [0b1, 0b11, 0b111, 0b1111, 0b11111])
    assert TR.depth_anc(TR.star(4)) == ([0, 1, 1, 1], [0b1, 0b11, 0b101, 0b1001])
    #        0
    #      1   2
    #     3 4   5
    d, a = TR.depth_anc([0, 0, 0, 1, 1, 2])
    assert d == [0, 1, 1, 2, 2, 2] and a == [0b1, 0b11, 0b101, 0b1011, 0b10011, 0b100101]
    # malformed parents (out of [0, t)) read as the root: the walk ends
    d, a = TR.depth_anc([7, 5, -1, 3])
    assert d == [0, 1, 1, 1] and a == [0b1, 0b11, 0b101, 0b1001]
    d, _ = TR.depth_anc(TR.deepest_last(8))
    assert d == [0, 1, 2, 3, 1, 2, 3, 4]


@pytest.mark.parametrize("T", [1, 2, 3, 5, 16])
def test_chain_mask_is_the_row_limit(T):
    for L in (T, T + 1, 64 + T, 300):
        assert TR.chain_limits_equal_mask(L, T)


@pytest.mark.parametrize("mode", [KV.QUANT_NONE, KV.QUANT_I8, KV.QUANT_U4])
@pytest.mark.parametrize("T", [1, 3, 4])
def test_chain_attention_equals_tokens_oracle(mode, T):
    rng = np.random.default_rng(11 + T + mode)
    nH, nG, span = 8, 2, 16
    lens = [T, 37, 70]
    kref, vref = KV.SpanCacheRef(mode, span, nG), KV.SpanCacheRef(mode, span, nG)
    for b, L in enumerate(lens):
        kref.add_sequence(); vref.add_sequence()
        for pos in range(L):
            kref.append(b, pos, rng.standard_normal((nG, 128)).astype(np.float32))
            vref.append(b, pos, rng.standard_normal((nG, 128)).astype(np.float32))
    q = rng.standard_normal((len(lens), T, nH, 128)).astype(np.float32)
    a = 1 / np.sqrt(128)
    got, got_abs = TR.attention_tree(q, kref, vref, lens, [TR.chain(T)] * len(lens), T, nH, a, with_abs=True)
    want, want_abs = S.attention_tokens(q, kref, vref, lens, T, nH, a, with_abs=True)
    assert np.array_equal(got, want) and np.array_equal(got_abs, want_abs)


def test_tree_attention_rows_see_only_ancestors():
    """a row equals the dense attention over the prefix plus its ancestors' slots"""
    rng = np.random.default_rng(3)
    nH, nG, span, T, L = 4, 1, 16, 6, 40
    par = [0, 0, 0, 1, 2, 4]
    kref, vref = KV.SpanCacheRef(KV.QUANT_NONE, span, nG), KV.SpanCacheRef(KV.QUANT_NONE, span, nG)
    kref.add_sequence(); vref.add_sequence()
    for pos in range(L):
        kref.append(0, pos, rng.standard_normal((nG, 128)).astype(np.float32))
        vref.append(0, pos, rng.standard_normal((nG, 128)).astype(np.float32))
    q = rng.standard_normal((1, T, nH, 128)).astype(np.float32)
    got = TR.attention_tree(q, kref, vref, [L], [par], T, nH, 1 / np.sqrt(128))
    K, V = kref.dense(0, L)[0].astype(np.float64), vref.dense(0, L)[0].astype(np.float64)
    _, anc = TR.depth_anc(par)
    for t in range(T):
        cols = list(range(L - T)) + [L - T + j for j in range(T) if anc[t] >> j & 1]
        for h in range(nH):
            s = (K[cols] @ q[0, t, h].astype(np.float64)) / np.sqrt(128)
            p = np.exp(s - s.max())
            np.testing.assert_allclose(got[0, t, h], (p / p.sum()) @ V[cols], rtol=1e-6, atol=1e-6)


def test_accept_chain_equals_spec_accept():
    rng = np.random.default_rng(5)
    for T in (1, 2, 4, 8, 16):
        B = 32
        pred = rng.integers(0, 3, (B, T))
        tokens = rng.integers(0, 3, (B, T))
        tokens[::4, 1:] = pred[::4, :-1]
        n, paths, nxt = TR.accept_tree(tokens, pred, [TR.chain(T)] * B)
        n_ref, nxt_ref = S.accept(tokens, pred)
        assert n.tolist() == n_ref.tolist() and nxt.tolist() == nxt_ref.tolist()
        assert all(p == list(range(k)) for p, k in zip(paths, n))


def test_accept_rule_hand_written_trees():
    # star: drafts 1..3 are all children of the root; the first one equal to pred[0] wins
    n, paths, nxt = TR.accept_tree([[10, 5, 11, 11]], [[11, 20, 21, 22]], [TR.star(4)])
    assert n.tolist() == [2] and paths == [[0, 2]] and nxt.tolist() == [21]
    # chain, all right
    n, paths, nxt = TR.accept_tree([[10, 11, 12, 13]], [[11, 12, 13, 14]], [TR.chain(4)])
    assert n.tolist() == [4] and paths == [[0, 1, 2, 3]] and nxt.tolist() == [14]
    # deep branch: root -> 1 (wrong) ; root -> 2 -> 3 -> 4 (right)
    par = [0, 0, 0, 2, 3]
    n, paths, nxt = TR.accept_tree([[10, 99, 11, 12, 13]], [[11, 7, 12, 13, 14]], [par])
    assert n.tolist() == [4] and paths == [[0, 2, 3, 4]] and nxt.tolist() == [14]
    # duplicate sibling tokens: both 1 and 2 match pred[0]; the lowest index is taken, even though 2's subtree goes deeper
    par = [0, 0, 0, 2]
    n, paths, nxt = TR.accept_tree([[10, 11, 11, 12]], [[11, 50, 12, 13]], [par])
    assert n.tolist() == [2] and paths == [[0, 1]] and nxt.tolist() == [50]
    # nothing right
    n, paths, nxt = TR.accept_tree([[10, 1, 2, 3]], [[9, 9, 9, 9]], [par])
    assert n.tolist() == [1] and paths == [[0]] and nxt.tolist() == [9]
    # the match must be a child of the current node: node 3 matches pred[0] but hangs below 2
    n, paths, _ = TR.accept_tree([[10, 4, 5, 11]], [[11, 0, 0, 0]], [par])
    assert n.tolist() == [1]


def _spans(mode, span, nG, n_spans, rng):
    nbytes = KV.span_bytes(mode if mode != 3 else KV.QUANT_I8, span, nG)
    return [rng.integers(0, 256, nbytes, dtype=np.uint8) for _ in range(n_spans)]


@pytest.mark.parametrize("mode", [0, 1, 2, 3])
def test_compaction_hazard_family(mode):
    """path [0, 2, 3, ...]: slot 2 is read for i = 1 and written for i = 2.  Sequential copies in increasing i equal a copy
    that reads every source row first; a copy in decreasing i (one schedule of a barrier-free parallel copy) differs."""
    rng = np.random.default_rng(mode)
    span, nG = 16, 2
    for base in (0, 13, 15):  # the path crosses a span edge from base 13 and 15
        for path in ([0, 2, 3], [0, 2, 3, 4], [0, 3, 5, 6], [0, 1, 3, 4]):
            spans = _spans(mode, span, nG, 3, rng)
            seq = [s.copy() for s in spans]
            TR.compact(seq, mode, span, nG, base, path)
            # read all sources, then write
            snap = [s.copy() for s in spans]
            first = [s.copy() for s in spans]
            for i in range(1, len(path)):
                if path[i] != i:
                    sa, ps = snap[(base + path[i]) // span], (base + path[i]) % span
                    da, pd = first[(base + i) // span], (base + i) % span
                    for g in range(nG):
                        for (s0, s1), (d0, d1) in zip(TR.row_ranges(mode, span, nG, g, ps), TR.row_ranges(mode, span, nG, g, pd)):
                            da[d0:d1] = sa[s0:s1]
            assert all(np.array_equal(a, b) for a, b in zip(seq, first))
            rev = [s.copy() for s in spans]
            TR.compact_in_order(rev, mode, span, nG, base, path, range(len(path) - 1, 0, -1))
            hazard = any(path[j] == i for i in range(1, len(path)) for j in range(1, i) if path[i] != i)
            assert hazard == (not all(np.array_equal(a, b) for a, b in zip(seq, rev))), path
            # slot base + i now holds what slot base + path[i] held
            for i in range(len(path)):
                for g in range(nG):
                    s, d = base + path[i], base + i
                    for (s0, s1), (d0, d1) in zip(TR.row_ranges(mode, span, nG, g, s % span), TR.row_ranges(mode, span, nG, g, d % span)):
                        assert np.array_equal(seq[d // span][d0:d1], spans[s // span][s0:s1])


def test_argument_checks_without_gpu():
    from b200spark import _lib
    lib = _lib.lib
    one = C.c_void_p(16)  # never dereferenced: the checks come first
    cfg = _lib.SpanCfg(_lib.DT_BF16, 0, 28, 4, 128, 16, 8, 0)
    cfg64 = _lib.SpanCfg(_lib.DT_BF16, 0, 14, 2, 64, 16, 8, 0)
    # NULL -> PARAM
    assert lib.b2_span_cache_append_tree(C.byref(cfg), one, one, one, one, one, None, 2, 4, None, None) == 3
    assert lib.b2_span_attn_run_tree(None, one, one, one, one, one, one, 2, 4, 64, one, 1 << 20, 1.0, None) == 3
    assert lib.b2_spec_accept_tree(one, None, one, one, one, one, one, one, 2, 4, None) == 3
    assert lib.b2_spec_accept_tree(one, one, one, one, one, one, one, None, 2, 4, None) == 3
    assert lib.b2_span_cache_compact(C.byref(cfg), one, one, 3, one, one, None, 2, 4, None) == 3
    assert lib.b2_span_cache_compact(C.byref(cfg), one, one, 0, one, one, one, 2, 4, None) == 3
    # q_len 0 / 17 -> LIMIT
    for T in (0, 17):
        assert lib.b2_span_cache_append_tree(C.byref(cfg), one, one, one, one, one, one, 2, T, None, None) == 4
        assert lib.b2_spec_accept_tree(one, one, one, one, one, one, one, one, 2, T, None) == 4
        assert lib.b2_span_cache_compact(C.byref(cfg), one, one, 3, one, one, one, 2, T, None) == 4
    # head 64 -> UNSUPPORTED
    assert lib.b2_span_cache_append_tree(C.byref(cfg64), one, one, one, one, one, one, 2, 4, None, None) == 6
    assert lib.b2_span_cache_compact(C.byref(cfg64), one, one, 3, one, one, one, 2, 4, None) == 6
