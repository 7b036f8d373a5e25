"""CPU restatement of sampled speculative verification (b2_sample_tokens + b2_spec_accept_sampled, include/b200spark.h).

Row (b, t) of a verify step is draft node t of sequence b.  It is drawn by b2_sample's rule (sample_ref.sample_row) with
sequence b's parameters at counter offsets[b] + depth(t) (tree_ref.depth_anc; t for a chain).  The walk is greedy
verification's over the draws (spec_ref.accept for a chain, tree_ref.accept_tree for a tree), and offsets[b] then
advances by the accepted count.

`Oracle` gives logits as a deterministic function of the token context, so a single-token sampling loop and a
speculative loop can be run over identical rows: their token streams and final offsets must be equal for any drafter.
`DRAFTERS` are the drafters the tests use; `variant` restates one wrong kernel each (MUTATIONS).  Imports without the
native library."""
import zlib

import numpy as np
import torch

import glue_ref as G
import sample_ref as SR
import spec_ref as S
import tree_ref as TR

MUTATIONS = ["node_counter", "advance_T", "advance_n_minus_1", "no_advance", "params_by_row", "row_in_counter",
             "highest_child", "compare_own"]
# the per-sequence parameters of the tests: sampled with top-k / top-p, plain, greedy (t = 0), hot with a small k
PARAMS = [(0.7, 50, 0.9), (1.0, 0, 1.0), (0.0, 0, 1.0), (1.3, 5, 0.8)]


# ------------------------------------------------------------------------------------------------------------- the step
def params_of(B, seed=0):
    """(temperature fp32 [B], top_k int32 [B], top_p fp32 [B], seeds uint64 [B]) cycling through PARAMS"""
    t = np.array([PARAMS[b % len(PARAMS)][0] for b in range(B)], np.float32)
    k = np.array([PARAMS[b % len(PARAMS)][1] for b in range(B)], np.int32)
    p = np.array([PARAMS[b % len(PARAMS)][2] for b in range(B)], np.float32)
    seeds = np.array([(0x9E3779B97F4A7C15 * (b + 1) + seed) % 2 ** 64 for b in range(B)], np.uint64)
    return t, k, p, seeds


def counters(offsets, parents, B, T, variant=None):
    """[B, T] uint64: the Philox counter of each row, offsets[b] + depth(t)"""
    out = np.zeros((B, T), np.uint64)
    for b in range(B):
        depth = list(range(T)) if parents is None else TR.depth_anc(parents[b])[0]
        for t in range(T):
            out[b, t] = (int(offsets[b]) + (t if variant == "node_counter" else depth[t])) % 2 ** 64
    return out


def sample_tokens(rows, T, params, offsets, parents=None, form="fp64", variant=None):
    """b2_sample_tokens on the host: rows fp32 [B*T, n]; returns the draws int64 [B, T] (offsets are not changed)"""
    t, k, p, seeds = params
    B = rows.shape[0] // T
    ctr = counters(offsets, parents, B, T, variant)
    pred = np.zeros((B, T), np.int64)
    for b in range(B):
        for u in range(T):
            r = b * T + u
            q = r % B if variant == "params_by_row" else b
            pred[b, u] = SR.sample_row(rows[r], t[q], k[q], p[q], seeds[q], ctr[b, u], row=r, form=form,
                                       variant="row_in_counter" if variant == "row_in_counter" else None)
    return pred


def _walk(tk, pr, par, variant):
    """one sequence's walk with a restated bug: the highest-index matching child, or tokens[c] compared with pred[c]"""
    T = len(tk)
    u, path = 0, [0]
    while True:
        kids = [c for c in range(u + 1, T) if TR.parent(par, c) == u
                and tk[c] == (pr[c] if variant == "compare_own" else pr[u])]
        if not kids:
            return path
        u = max(kids) if variant == "highest_child" else min(kids)
        path.append(u)


def accept(tokens, pred, parents=None, variant=None):
    """the walk of b2_spec_accept_sampled: (accepted [B], paths (lists), next_ids [B])"""
    tokens, pred = np.asarray(tokens), np.asarray(pred)
    B, T = tokens.shape
    if variant in ("highest_child", "compare_own"):
        pars = [TR.chain(T)] * B if parents is None else parents
        paths = [_walk(tokens[b], pred[b], pars[b], variant) for b in range(B)]
        n = np.array([len(pa) for pa in paths], np.int64)
        return n, paths, np.array([pred[b, pa[-1]] for b, pa in enumerate(paths)], np.int64)
    if parents is None:
        n, nxt = S.accept(tokens, pred)
        return n, [list(range(int(v))) for v in n], nxt
    return TR.accept_tree(tokens, pred, parents)


def advance(offsets, accepted, T, variant=None):
    """the offsets after the step"""
    d = {"advance_T": np.full_like(accepted, T), "advance_n_minus_1": accepted - 1,
         "no_advance": np.zeros_like(accepted)}.get(variant, accepted)
    return np.asarray(offsets, np.uint64) + d.astype(np.uint64)


def step(rows, tokens, params, offsets, parents=None, form="fp64", variant=None):
    """one sampled verify step: (pred [B, T], accepted [B], paths, next_ids [B], offsets after)"""
    T = tokens.shape[1]
    pred = sample_tokens(rows, T, params, offsets, parents, form, variant)
    n, paths, nxt = accept(tokens, pred, parents, variant)
    return pred, n, paths, nxt, advance(offsets, n, T, variant)


# ------------------------------------------------------------------------------------------------------------- the oracle
class Oracle:
    """Logits that are a deterministic function of the token context (every token so far), rounded to dt.  Three rows in
    four are peaked (one token well above a few runners-up and an N(0, 1) floor), so a drafter that knows the likely
    continuation is often right; the fourth is a flat N(0, 2) row."""

    def __init__(self, vocab, seed=0, dt=torch.bfloat16, perturb=0.0):
        self.vocab, self.seed, self.dt, self.perturb = vocab, seed, dt, perturb
        self.cache = {}

    def row(self, ctx):
        key = tuple(int(v) for v in ctx)
        if key not in self.cache:
            h = zlib.crc32(np.asarray(key, np.int64).tobytes(), self.seed)
            rng = np.random.default_rng([self.seed, h, len(key)])
            kind = h % 4
            x = rng.standard_normal(self.vocab) * (2.0 if kind == 3 else 1.0)
            if kind < 3:
                top = rng.choice(self.vocab, 4, replace=False)
                x[top] = [[14.0, 9.0, 8.5, 8.0], [10.0, 9.5, 9.0, 7.0], [8.0, 7.5, 7.0, 6.5]][kind]
            if self.perturb:  # a draft model's view of the same row
                x = x + np.random.default_rng([self.seed + 1, h]).standard_normal(self.vocab) * self.perturb
            self.cache[key] = G.ft_values(x, self.dt)
        return self.cache[key]


def contexts(ctx, tokens, par):
    """the contexts of a sequence's T nodes: ctx (ending with the last emitted token, node 0) plus the drafts on the path
    from the root to the node"""
    out = []
    for t in range(len(tokens)):
        path, u = [], t
        while u > 0:
            path.append(int(tokens[u]))
            u = TR.parent(par, u)
        out.append(list(ctx) + path[::-1])
    return out


# ------------------------------------------------------------------------------------------------------------- trees and drafters
def topk_tree(T):
    """each node's children are its parent's most likely tokens: 3 below the root, 2 below each depth-1 node, then 1"""
    par, frontier, fan = [0], [0], [3, 2]
    while len(par) < T:
        nxt = []
        for u in frontier:
            depth = TR.depth_anc(par)[0][u]
            for _ in range(fan[depth] if depth < len(fan) else 1):
                if len(par) < T:
                    par.append(u)
                    nxt.append(len(par) - 1)
        frontier = nxt
    return par


TREES = {"chain": lambda rng, T: TR.chain(T), "star": lambda rng, T: TR.star(T), "random_tree": TR.random_tree,
         "deepest_last": lambda rng, T: TR.deepest_last(T), "topk": lambda rng, T: topk_tree(T)}


def draft(kind, rng, oracle, ctx, par, truth=None, draft_oracle=None):
    """draft tokens [T] for nodes 1.. (node 0 = ctx[-1]) in node order, so a node's context is known when it is drafted.
    random: uniform ids.  truth: the true continuation at the node's depth (truth[d - 1]; random past its end), one in four corrupted.
    argmax: the parent row's argmax; in a topk tree, the parent row's i-th most likely token for its i-th child.
    sampled: a draw from draft_oracle's row of the parent context (its own seed and counter)."""
    T = len(par)
    tokens = np.zeros(T, np.int64)
    tokens[0] = ctx[-1]
    depth = TR.depth_anc(par)[0]
    rank = {}
    for c in range(1, T):
        u = TR.parent(par, c)
        pctx = contexts(ctx, tokens[:u + 1], par[:u + 1])[u]
        if kind == "random":
            tokens[c] = rng.integers(0, oracle.vocab)
        elif kind == "truth":
            right = depth[c] <= len(truth) and rng.random() >= 0.25
            tokens[c] = truth[depth[c] - 1] if right else rng.integers(0, oracle.vocab)
        elif kind == "argmax":
            i = rank.get(u, 0)
            rank[u] = i + 1
            tokens[c] = SR.order(oracle.row(pctx))[i]
        else:
            tokens[c] = SR.sample_row(draft_oracle.row(pctx), 1.0, 0, 1.0, 12345, len(pctx), form="fp64")
    return tokens


DRAFTERS = ["random", "truth", "argmax", "sampled"]


# ------------------------------------------------------------------------------------------------------------- the loops
def sample_stream(oracle, prompt, params, b, off, L, form="fp64"):
    """single-token sampling of sequence b for L tokens (b2_sample at counters off, off + 1, ...)"""
    t, k, p, seeds = params
    ctx, out = list(prompt), []
    for _ in range(L):
        out.append(SR.sample_row(oracle.row(ctx), t[b], k[b], p[b], seeds[b], off + len(out), form=form))
        ctx.append(out[-1])
    return out, off + L


def spec_stream(oracle, prompts, params, offsets, L, T, tree, drafter, seed=0, truths=None, variant=None, form="fp64"):
    """the speculative loop: verify steps of T rows per sequence until every sequence has at least L tokens.  Returns
    (tokens per sequence, offsets, accepted counts per step)"""
    rng = np.random.default_rng(seed)
    B = len(prompts)
    ctx = [list(pr) for pr in prompts]
    out = [[] for _ in range(B)]
    off = np.asarray(offsets, np.uint64).copy()
    dor = Oracle(oracle.vocab, oracle.seed, oracle.dt, perturb=0.7) if drafter == "sampled" else None
    counts = []
    while min(len(o) for o in out) < L:
        pars = [TREES[tree](rng, T) for _ in range(B)]
        tokens = np.stack([draft(drafter, rng, oracle, ctx[b], pars[b], None if truths is None else truths[b][len(out[b]):],
                                 dor) for b in range(B)])
        rows = np.stack([oracle.row(c) for b in range(B) for c in contexts(ctx[b], tokens[b], pars[b])])
        parents = None if tree == "chain" else np.asarray(pars, np.int32)
        pred, n, paths, _, off = step(rows, tokens, params, off, parents, form, variant)
        for b in range(B):
            emitted = [int(pred[b, u]) for u in paths[b]]
            out[b] += emitted
            ctx[b] += emitted
        counts.append(n)
    return out, off, counts
