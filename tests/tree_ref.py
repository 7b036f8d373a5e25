"""CPU restatements of tree-structured speculative verification: depth / ancestor masks from parents, attention with
per-row ancestor masks, the greedy tree accept rule of b2_spec_accept_tree and the compaction of b2_span_cache_compact on
span bytes.  Tree format: include/b200spark.h (parents[t] in [0, t) for t >= 1; node 0 is the root).  Imports without
the native library."""
import numpy as np

import spec_ref as S

ROW_BYTES = {0: 256, 1: 128, 2: 64, 3: 128}  # KV mode -> bytes per token row (none / i8 / u4 / fp8; KVTraits::ROW)


# ------------------------------------------------------------------------------------------------------------- trees
def parent(par, t):
    """The parent the kernels use (tree_parent): par[t] when it lies in [0, t), else the root."""
    p = int(par[t])
    return p if 0 <= p < t else 0


def depth_anc(par):
    """par [T] -> (depth [T], anc [T]): parent steps to node 0, and the bit mask of t and its ancestors."""
    T = len(par)
    depth, anc = [0] * T, [0] * T
    for t in range(T):
        u, a, d = t, 1 << t, 0
        while u > 0:
            u = parent(par, u)
            a |= 1 << u
            d += 1
        depth[t], anc[t] = d, a
    return depth, anc


def chain(T):
    return [0] + list(range(T - 1))


def star(T):
    """every draft a child of the root"""
    return [0] * T


def random_tree(rng, T):
    return [0] + [int(rng.integers(0, t)) for t in range(1, T)]


def deepest_last(T):
    """a root with a short branch and, last, the deepest one: nodes 1 .. T//2 - 1 a chain off the root, the rest another"""
    h = max(1, T // 2)
    return [0] + [0 if t in (1, h) else t - 1 for t in range(1, T)]


def tree_mask(L, par):
    """[T, L] visibility of a sequence of new length L whose last T slots hold the tree's nodes"""
    T = len(par)
    _, anc = depth_anc(par)
    pe = L - T
    mask = np.zeros((T, L), bool)
    mask[:, :pe] = True
    for t in range(T):
        for j in range(T):
            if anc[t] >> j & 1:
                mask[t, pe + j] = True
    return mask


# ------------------------------------------------------------------------------------------------------------- attention
def attention_tree(q, kcache, vcache, new_lens, parents, q_len, n_heads, alpha, with_abs=False):
    """q fp32 [B, q_len, nH, 128]; kcache / vcache: oracle.kvcache_ref.SpanCacheRef (or anything with .dense / .n_groups /
    .head); parents [B][q_len].  fp64 attention where row (b, t) sees the prefix and its ancestors' slots (tree_mask).  The
    arithmetic is spec_ref.attention_tokens' with the mask replaced, so a chain gives its results exactly.  Returns fp32
    [B, q_len, nH, 128]; with_abs: also sum_j p_j |V_j|."""
    B = q.shape[0]
    G = kcache.n_groups
    hpg = n_heads // G
    out = np.zeros((B, q_len, n_heads, kcache.head), np.float32)
    out_abs = np.zeros_like(out)
    for b in range(B):
        L = int(new_lens[b])
        K = kcache.dense(b, L).astype(np.float64)
        V = vcache.dense(b, L).astype(np.float64)
        mask = tree_mask(L, parents[b])
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


def chain_limits_equal_mask(L, T):
    """the chain's tree mask is spec_ref's per-row limit"""
    lim = np.array([S.row_limit(L, T, t) for t in range(T)])
    return np.array_equal(tree_mask(L, chain(T)), np.arange(L)[None, :] < lim[:, None])


# ------------------------------------------------------------------------------------------------------------- accept
def accept_tree(tokens, pred, parents):
    """b2_spec_accept_tree on the host: tokens / pred / parents [B, T].  Returns (accepted [B], paths (list of lists),
    next_ids [B])."""
    tokens, pred, parents = np.asarray(tokens), np.asarray(pred), np.asarray(parents)
    B, T = tokens.shape
    n, paths, nxt = np.ones(B, np.int64), [], np.zeros(B, np.int64)
    for b in range(B):
        u, path = 0, [0]
        while True:
            kids = [c for c in range(u + 1, T) if parent(parents[b], c) == u and tokens[b, c] == pred[b, u]]
            if not kids:
                break
            u = min(kids)
            path.append(u)
        n[b], nxt[b] = len(path), pred[b, u]
        paths.append(path)
    return n, paths, nxt


# ------------------------------------------------------------------------------------------------------------- compaction
def row_ranges(mode, span_len, n_groups, g, pos):
    """byte ranges of (kv-head g, in-span position pos) in a span: the row, then its {zero, scale} (quantized modes)"""
    R = ROW_BYTES[mode]
    r = g * span_len + pos
    out = [(r * R, (r + 1) * R)]
    if mode != 0:
        p0 = n_groups * span_len * R + r * 8
        out.append((p0, p0 + 8))
    return out


def _slot(spans, span_len, s):
    return spans[s // span_len], s % span_len


def copy_slot(spans, mode, span_len, n_groups, src, dst):
    """copy slot src to slot dst for every kv-head (spans: one sequence's list of uint8 span arrays, modified in place)"""
    sa, ps = _slot(spans, span_len, src)
    da, pd = _slot(spans, span_len, dst)
    for g in range(n_groups):
        for (s0, s1), (d0, d1) in zip(row_ranges(mode, span_len, n_groups, g, ps), row_ranges(mode, span_len, n_groups, g, pd)):
            da[d0:d1] = sa[s0:s1].copy()


def compact(spans, mode, span_len, n_groups, base, path):
    """b2_span_cache_compact for one sequence and one of K / V: slot base + path[i] -> base + i, 1 <= i < len(path), in
    increasing i (each source is read before any later copy could write it: path[i] >= i)."""
    for i in range(1, len(path)):
        if path[i] != i:
            copy_slot(spans, mode, span_len, n_groups, base + path[i], base + i)


def compact_in_order(spans, mode, span_len, n_groups, base, path, order):
    """the same copies, each read right before its write, in the given order of i: what a copy that runs every i in
    parallel without a barrier can produce"""
    for i in order:
        if path[i] != i:
            copy_slot(spans, mode, span_len, n_groups, base + path[i], base + i)
