"""CPU restatement of b2_penalize_tokens (include/b200spark.h), by construction: for every row (b, t) of a verify step,
build the virtual history V(b, t) (slot b followed by the drafts on the path from the root to node t, appended with
penalty_ref.History's semantics: ids outside [0, vocab) become -1, appends stop at max_len, the prompt length stays) and
run penalty_ref.penalize on it.

`bugs` restates one wrong processor each (BUGS); the CPU suite shows that every one of them changes an output.  Imports
without the native library."""
import numpy as np

import penalty_ref as P
import tree_ref as TR

BUGS = ["root_appended", "lower_nodes", "own_left_out", "path_as_prompt", "duplicate_once", "min_len_base",
        "ngram_base_only", "max_len_ignored", "oob_as_itself"]


def path_nodes(parents, t, bugs=()):
    """the non-root nodes on the path from the root to t, ascending (parents None: a chain, nodes 1 .. t)"""
    if parents is None or "lower_nodes" in bugs:
        nodes = list(range(1, t + 1))
    else:
        anc = TR.depth_anc(parents)[1][t]
        nodes = [u for u in range(1, t + 1) if anc >> u & 1]
    if "root_appended" in bugs:
        nodes = [0] + nodes
    if "own_left_out" in bugs:
        nodes = [u for u in nodes if u != t]
    return nodes


def virtual(base, prompt_len, row, parents, t, max_len, vocab, bugs=()):
    """V(b, t) as (tokens, prompt length): base = slot b's stored tokens (-1 for ids outside the vocabulary), row = the
    sequence's draft tokens [T] (row[0] = the last emitted token, never appended)"""
    h = P.History(1, max_len + (1 << 20 if "max_len_ignored" in bugs else 0), vocab)
    h.tokens[0] = [int(v) for v in base]
    h.prompt[0] = prompt_len
    path = [int(row[u]) for u in path_nodes(parents, t, bugs)]
    if "duplicate_once" in bugs:
        path = [v for i, v in enumerate(path) if v not in path[:i]]
    for v in path:
        if "oob_as_itself" in bugs:
            if len(h.tokens[0]) < h.max_len:
                h.tokens[0].append(v)
        else:
            h.append([v])
    return h.tokens[0], (len(h.tokens[0]) if "path_as_prompt" in bugs else prompt_len)


def ngram_bans(hist, g):
    """the ids the no-repeat n-gram step bans over hist (g == 1: every id of it)"""
    L = len(hist)
    if g == 1:
        return [t for t in hist if t >= 0]
    return [hist[j + g - 1] for j in range(0, L - g + 1) if g > 1 and hist[j:j + g - 1] == hist[L - g + 1:L]]


def penalize_tokens(x, hists, prompts, tokens, parents, params, ft, max_len, vocab, id_offset=0, bugs=()):
    """x: fp64 [B*T, n] FT values of vocabulary ids [id_offset, id_offset + n); hists: B stored base histories; prompts [B];
    tokens [B][T]; parents None (chains) or [B][T]; params: per-sequence lists (penalty_ref.penalize's keys).  Returns
    (out, alt) as penalty_ref.penalize does."""
    bugs = set(bugs)
    B = len(hists)
    T = len(tokens[0])
    rows, lens, plens = [], [], []
    prm = {k: [] for k in params}
    for b in range(B):
        for t in range(T):
            V, pl = virtual(hists[b], prompts[b], tokens[b], None if parents is None else parents[b], t, max_len, vocab, bugs)
            rows.append(V)
            lens.append(len(V))
            plens.append(pl)
            for k in params:
                prm[k].append(params[k][b])
            if "min_len_base" in bugs:  # compare against L instead of L'
                prm["min_length"][-1] += len(V) - len(hists[b])
            if "ngram_base_only" in bugs:
                prm["no_repeat_ngram"][-1] = 0
    tok = np.full((B * T, max(1, max(lens))), -1, np.int64)
    for r, V in enumerate(rows):
        tok[r, :len(V)] = V
    out, alt = P.penalize(x, tok, lens, plens, prm, ft, id_offset)
    if "ngram_base_only" in bugs:
        n = x.shape[1]
        ban = P.rn(P.BAN, ft)[()]
        for r in range(B * T):
            for v in ngram_bans([int(u) for u in hists[r // T]], int(params["no_repeat_ngram"][r // T])):
                if 0 <= v - id_offset < n:
                    out[r, v - id_offset] = alt[r, v - id_offset] = ban
    return out, alt


def virtual_rows(hists, prompts, tokens, parents, max_len, vocab):
    """every V(b, t) as (tokens, prompt length), row order b * T + t"""
    T = len(tokens[0])
    return [virtual(hists[b], prompts[b], tokens[b], None if parents is None else parents[b], t, max_len, vocab)
            for b in range(len(hists)) for t in range(T)]
