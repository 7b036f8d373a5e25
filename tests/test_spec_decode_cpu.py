"""CPU: the multi-token decode step's oracle, accept rule and work split (tests/spec_ref.py), and the argument checks of
the multi-token entry points that fail before touching the device."""
import ctypes as C
from collections import Counter

import numpy as np
import pytest

import attn_needles as A
import spec_ref as S
from oracle import kvcache_ref as KV


@pytest.mark.parametrize("mode", [KV.QUANT_NONE, KV.QUANT_I8, KV.QUANT_U4])
@pytest.mark.parametrize("T", [1, 3, 4])
def test_oracle_equals_single_token_calls(mode, T):
    """Row t of the multi-token oracle is attention_ref at length new_len - T + 1 + t."""
    rng = np.random.default_rng(7 + T + mode)
    nH, nG, span = 8, 2, 16
    lens = [T, 37, 70]
    kref, vref = KV.SpanCacheRef(mode, span, nG), KV.SpanCacheRef(mode, span, nG)
    for b, L in enumerate(lens):
        kref.add_sequence(); vref.add_sequence()
        for pos in range(L):
            kref.append(b, pos, rng.standard_normal((nG, 128)).astype(np.float32))
            vref.append(b, pos, rng.standard_normal((nG, 128)).astype(np.float32))
    q = rng.standard_normal((len(lens), T, nH, 128)).astype(np.float32)
    got = S.attention_tokens(q, kref, vref, lens, T, nH, 1 / np.sqrt(128))
    for t in range(T):
        want = KV.attention_ref(q[:, t], kref, vref, [L - T + 1 + t for L in lens], nH, 1 / np.sqrt(128))
        np.testing.assert_allclose(got[:, t], want, rtol=1e-6, atol=1e-6)


def test_accept_rule_cases():
    # tokens[b][0] = last emitted, tokens[b][1..] = drafts; pred[b][i] = the model's token after tokens[b][..i]
    pred = np.array([[11, 12, 13, 14]] * 4)
    tokens = np.array([[10, 11, 12, 13],   # all drafts right
                       [10, 99, 12, 13],   # first draft wrong
                       [10, 11, 99, 13],   # middle draft wrong
                       [10, 11, 12, 99]])  # last draft wrong
    n, nxt = S.accept(tokens, pred)
    assert n.tolist() == [4, 1, 2, 3]
    assert nxt.tolist() == [14, 11, 12, 13]
    n, nxt = S.accept(np.array([[5], [6]]), np.array([[7], [8]]))  # T = 1: plain greedy decoding
    assert n.tolist() == [1, 1] and nxt.tolist() == [7, 8]
    # a later match after a mismatch does not count
    n, _ = S.accept(np.array([[1, 9, 3, 4]]), np.array([[2, 3, 4, 5]]))
    assert n.tolist() == [1]


@pytest.mark.parametrize("hpg", [1, 4, 7, 8, 16])
@pytest.mark.parametrize("T", [1, 2, 3, 4, 8, 16])
def test_row_blocks(hpg, T):
    tpb, nrb = S.row_blocks(hpg, T)
    assert 1 <= tpb <= T and tpb * hpg <= 16 and nrb * tpb >= T and (nrb - 1) * tpb < T


@pytest.mark.parametrize("seed", range(6))
def test_work_split_covers_every_tile_once(seed):
    rng = np.random.default_rng(seed)
    for _ in range(20):
        T = int(rng.choice([1, 2, 3, 4, 8, 16]))
        hpg = int(rng.choice([1, 4, 7, 8, 16]))
        nG = int(rng.choice([1, 2, 4]))
        B = int(rng.integers(1, 9))
        lens = [int(rng.integers(T, 2050)) for _ in range(B)]
        grid = int(rng.choice([1, 7, 132, 396]))
        cap = rng.choice([None, 1, 4, 17])
        dec = S.decompose_tokens(lens, T, hpg, nG, grid, None if cap is None else int(cap))
        A.check_decomposition(dec, S.block_lens(lens, T, hpg))
        tpb, nrb = S.row_blocks(hpg, T)
        want = Counter()
        for b, L in enumerate(lens):
            for rb in range(nrb):
                last = min(T, (rb + 1) * tpb) - 1
                for g in range(nG):
                    for tile in range(-(-S.row_limit(L, T, last) // 64)):
                        want[(b, rb, g, tile)] += 1
        assert Counter(S.tiles_covered(dec, lens, T, hpg)) == want


def test_argument_checks_without_gpu():
    from b200spark import _lib
    lib = _lib.lib
    one = C.c_void_p(16)  # never dereferenced: the checks come first
    cfg = _lib.SpanCfg(_lib.DT_BF16, 0, 28, 4, 128, 16, 8, 0)
    for T in (0, 17):
        assert lib.b2_span_cache_append_tokens(C.byref(cfg), one, one, one, one, one, 2, T, None, None) == 4
        assert lib.b2_spec_accept(one, one, one, one, one, one, 2, T, None) == 4
    cfg64 = _lib.SpanCfg(_lib.DT_BF16, 0, 14, 2, 64, 16, 8, 0)
    assert lib.b2_span_cache_append_tokens(C.byref(cfg64), one, one, one, one, one, 2, 4, None, None) == 6
    assert lib.b2_span_attn_run_tokens(None, one, one, one, one, one, 2, 4, 64, one, 1 << 20, 1.0, None) == 3
    assert lib.b2_span_attn_tokens_workspace_bytes(None, 2, 4, 64) == 0
