"""CPU restatements of the multi-token decode step (speculative decoding): attention with a per-row causal limit, the
greedy accept rule of b2_spec_accept and the (sequence, row block, kv-head, tile) work split of the multi-token
span_attn_kernel.  Imports without the native library."""
import numpy as np

import attn_needles as A

MAX_Q_LEN = 16


def row_blocks(hpg, q_len):
    """Whole tokens per block of 16 MMA rows: (tokens per block, blocks per sequence)."""
    tpb = min(q_len, 16 // hpg)
    return tpb, -(-q_len // tpb)


def row_limit(new_len, q_len, t):
    """Tokens row t of a q_len-token step attends to: itself and the tokens before it."""
    return new_len - q_len + 1 + t


def block_lens(lens, q_len, hpg):
    """Per (sequence, row block) item: the tokens its last token sees (what the kernel streams)."""
    tpb, nrb = row_blocks(hpg, q_len)
    return [L - q_len + min(q_len, (rb + 1) * tpb) for L in lens for rb in range(nrb)]


def attention_tokens(q, kcache, vcache, new_lens, q_len, n_heads, alpha, with_abs=False):
    """q fp32 [B, q_len, nH, 128]; kcache / vcache: oracle.kvcache_ref.SpanCacheRef.  fp64 attention where row (b, t) is
    masked at row_limit(new_lens[b], q_len, t).  Returns fp32 [B, q_len, nH, 128]; with_abs: also sum_j p_j |V_j| (the
    scale of the error the rounding of the probabilities can cause)."""
    B = q.shape[0]
    G = kcache.n_groups
    hpg = n_heads // G
    out = np.zeros((B, q_len, n_heads, kcache.head), np.float32)
    out_abs = np.zeros_like(out)
    for b in range(B):
        L = int(new_lens[b])
        K = kcache.dense(b, L).astype(np.float64)
        V = vcache.dense(b, L).astype(np.float64)
        lim = np.array([row_limit(L, q_len, t) for t in range(q_len)])
        mask = np.arange(L)[None, :] < lim[:, None]  # [q_len, L]
        for h in range(n_heads):
            g = h // hpg
            s = alpha * (q[b, :, h].astype(np.float64) @ K[g].T)  # [q_len, L]
            s = np.where(mask, s, -np.inf)
            s = s - s.max(axis=1, keepdims=True)
            p = np.exp(s)
            p = p / p.sum(axis=1, keepdims=True)
            out[b, :, h] = (p @ V[g]).astype(np.float32)
            out_abs[b, :, h] = (p @ np.abs(V[g])).astype(np.float32)
    return (out, out_abs) if with_abs else out


def accept(tokens, pred):
    """b2_spec_accept on the host: tokens / pred int [B, T].  Returns (accepted [B], next_ids [B])."""
    tokens, pred = np.asarray(tokens), np.asarray(pred)
    B, T = tokens.shape
    n = np.ones(B, np.int64)
    for b in range(B):
        while n[b] < T and tokens[b, n[b]] == pred[b, n[b] - 1]:
            n[b] += 1
    return n, pred[np.arange(B), n - 1]


def decompose_tokens(lens, q_len, hpg, n_groups, grid, max_pieces=None):
    """The split the multi-token kernel derives on the device: the single-token split (attn_needles.decompose) over the
    (sequence, row block) items of block_lens, in sequence-major, then row-block order."""
    return A.decompose(block_lens(lens, q_len, hpg), n_groups, grid, max_pieces)


def tiles_covered(dec, lens, q_len, hpg):
    """Multiset of (sequence, row block, kv-head, tile) the pieces of a decomposition cover."""
    _, nrb = row_blocks(hpg, q_len)
    out = []
    for bg in dec.bgs:
        b, rb = divmod(bg.b, nrb)
        for pc in bg.pieces:
            for tile in range(pc.tile_lo - bg.start, pc.tile_hi - bg.start):
                out.append((b, rb, bg.g, tile))
    return out
