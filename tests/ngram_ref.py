"""CPU restatement of b2_ngram_draft and b2_history_append_tokens (include/b200spark.h), in plain Python over lists.

The drafter is restated from the contract: every end position's match length, the candidates, their periodic
continuations and the breadth-first trie.  The append is restated through tests/penalty_ref.History, one token at a time,
so it is b2_history_append's bookkeeping by construction.

`bugs` restates one wrong drafter or append each (BUGS); tests/test_ngram_draft_cpu.py shows that every one of them
changes an output, so the GPU comparison against the restatement would catch it in the kernel."""
import penalty_ref as P

BUGS = ["least_recent", "shorter_n", "self_match", "period_off_by_one", "truncate", "depth_first", "latest_candidate",
        "padding_below_last", "append_chain_index", "append_last_twice"]


def match_len(S, e, n_max):
    """m(e): the leading i < n_max with e - i >= 0 and S[e-i] == S[L-1-i]"""
    L, i = len(S), 0
    while i < n_max and e - i >= 0 and S[e - i] == S[L - 1 - i]:
        i += 1
    return i


def candidates(S, n_min, n_max, width, bugs=()):
    """the end positions of the drafts' matches, most recent first ([] without a match)"""
    L = len(S)
    ends = range(L if "self_match" in bugs else L - 1)  # e in [0, L-2]
    m = {e: match_len(S, e, n_max) for e in ends}
    if not m:
        return []
    nstar = max(m.values())
    if nstar < n_min:
        return []
    need = n_min if "shorter_n" in bugs else nstar
    hits = [e for e in ends if m[e] >= need]
    return hits[:width] if "least_recent" in bugs else hits[::-1][:width]


def continuation(S, e, n, bugs=()):
    """c_k = S[e+1 + (k mod p)], p = L-1-e, for k < n (positions past the history read as -1 in the bugs that reach them)"""
    L = len(S)
    p = L - e if "period_off_by_one" in bugs else max(L - 1 - e, 1)
    at = lambda i: S[i] if i < L else -1  # noqa: E731
    if "truncate" in bugs:
        return [S[e + 1 + k] for k in range(n) if e + 1 + k < L]
    return [at(e + 1 + k % p) for k in range(n)]


def trie(conts, q_len, bugs=()):
    """(tokens of nodes 1 .., parents of nodes 1 ..) of the first q_len nodes of the candidates' trie (a -1 token stays -1
    here).  Breadth first; within a level by parent index, then by the rank of the first candidate."""
    rank = {}  # prefix -> [first rank, last rank]
    kids = {(): []}
    for j, c in enumerate(conts):
        for d in range(1, len(c) + 1):
            pre = tuple(c[:d])
            if pre not in rank:
                rank[pre] = [j, j]
                kids[pre[:-1]].append(pre)
                kids[pre] = []
            rank[pre][1] = j
    key = (lambda pre: rank[pre][1]) if "latest_candidate" in bugs else (lambda pre: rank[pre][0])
    order = []
    if "depth_first" in bugs:
        def visit(pre):
            order.append(pre)
            for ch in sorted(kids[pre], key=key):
                visit(ch)
        visit(())
    else:
        level = [()]
        while level:
            order += level
            level = [ch for pre in level for ch in sorted(kids[pre], key=key)]
    order = order[:q_len]
    num = {pre: t for t, pre in enumerate(order)}
    return [pre[-1] for pre in order[1:]], [num[pre[:-1]] for pre in order[1:]]


def draft(S, tok0, q_len, n_min, n_max, width, tree, bugs=()):
    """One sequence: (tokens [q_len] with tokens[0] = tok0, parents [q_len] or None, n_draft)"""
    S = [int(t) for t in S]
    return draft_from(S, candidates(S, n_min, n_max, width, bugs), tok0, q_len, tree, bugs)


def draft_from(S, cands, tok0, q_len, tree, bugs=()):
    """draft() from the candidates (most recent first); candidates(S, n_min, n_max, w) is the first w of those for any
    larger width, so a caller may find them once for every width"""
    conts = [continuation(S, e, q_len - 1, bugs) for e in cands]
    fix = lambda t: tok0 if t == -1 else t  # noqa: E731
    if not tree:
        c = conts[0] if conts else []
        return [tok0] + [fix(t) for t in c] + [tok0] * (q_len - 1 - len(c)), None, len(c)
    toks, pars = trie(conts, q_len, bugs)
    nodes = 1 + len(toks)
    pad_par = (lambda t: t - 1) if "padding_below_last" in bugs else (lambda t: 0)
    tokens = [tok0] + [fix(t) for t in toks] + [tok0] * (q_len - nodes)
    parents = [0] + pars + [pad_par(t) for t in range(nodes, q_len)]
    return tokens, parents, nodes - 1


def draft_batch(hists, tok0, q_len, n_min, n_max, width, tree, bugs=()):
    """hists: per-sequence token lists (the history slots); tok0: column 0 per sequence.  Returns (tokens [B][q_len],
    parents [B][q_len] or None, n_draft [B])."""
    out = [draft(S, int(t), q_len, n_min, n_max, width, tree, bugs) for S, t in zip(hists, tok0)]
    return [o[0] for o in out], ([o[1] for o in out] if tree else None), [o[2] for o in out]


def emitted(pred, accepted, path=None, bugs=()):
    """the emitted tokens of a verify step per sequence: pred[b][path[b][i]] (chain: pred[b][i]) for i < accepted[b]"""
    chain = path is None or "append_chain_index" in bugs
    return [[int(pred[b][i if chain else path[b][i]]) for i in range(int(accepted[b]))] for b in range(len(accepted))]


def append_tokens(hist, pred, accepted, path=None, bugs=()):
    """b2_history_append_tokens on a penalty_ref.History: each emitted token through History.append of its own slot"""
    for b, ids in enumerate(emitted(pred, accepted, path, bugs)):
        if "append_last_twice" in bugs and hist.tokens[b]:
            ids = [hist.tokens[b][-1]] + ids
        one = P.History.__new__(P.History)  # a one-slot view of slot b (the token list is shared)
        one.rows, one.max_len, one.vocab, one.tokens, one.prompt = 1, hist.max_len, hist.vocab, [hist.tokens[b]], [0]
        for t in ids:
            one.append([t])
    return hist
