"""CPU restatement of b2_sample_shard / b2_sample_shard_merge (include/b200spark.h): b2_sample under tensor parallelism,
over numpy records.

A row of n_total columns is split into contiguous shards, rank q holding [bounds[q], bounds[q + 1]).  Each phase builds
every rank's record from its shard and the all-gathered records of the phase before, as the kernels do: the shard argmax
(phase 0), the level-1 histogram of the 16-bit order key's high byte at the row's m and c (1), the level-2 counts of the
pending selection's high byte (2, 3, 4), the holder's id (5).  `shard_sample_row` returns the merged id; on exact rows
(tests/sample_ref.py) it must equal `sample_row` for any split.

`variant` restates one wrong protocol each (MUTATIONS); the CPU suite shows that every one of them changes a drawn id on
crafted rows."""
import numpy as np
import torch

import sample_ref as S

MUTATIONS = ["shard_max", "topk_per_shard", "tie_high_rank", "no_prefix", "drop_offset", "u_rank_sp"]


def keys_of(x, dt):
    """the 16-bit order key of each value of x (representable in dt): the FT bits made order-preserving, -0 as +0"""
    b = torch.from_numpy(np.asarray(x, np.float32)).to(dt).view(torch.int16).numpy().astype(np.int64) & 0xFFFF
    b = np.where(b == 0x8000, 0, b)
    return np.where(b & 0x8000, ~b & 0xFFFF, b | 0x8000)


def scan(cnt, mass, by_mass, T):
    """smp_scan: the first bin from 255 down at which the running count (or weight) reaches T, and the counts / weights
    of the bins above it"""
    ac = am = 0
    for b in range(255, -1, -1):
        if (am + int(mass[b]) if by_mass else ac + int(cnt[b])) >= T or b == 0:
            return b, ac, am
        ac += int(cnt[b])
        am += int(mass[b])


def random_bounds(n, P, rng, one_col=False):
    """P contiguous shards of [0, n), each >= 1 column, unequal; one of them a single column when one_col"""
    assert 1 <= P <= n
    cuts = set()
    if one_col and P > 1:
        s = int(rng.integers(0, n))
        cuts |= {c for c in (s, s + 1) if 0 < c < n}
    while len(cuts) < P - 1:
        cuts.add(int(rng.integers(1, n)))
    return [0] + sorted(cuts)[:P - 1] + [n]


def even_bounds(n, P):
    """the decode stack's split: P equal shards (n divisible by P), or the last shard taking the remainder"""
    s = n // P
    return [q * s for q in range(P)] + [n]


def shard_sample_row(x, bounds, t, k, p, seed, off, dt=torch.bfloat16, form="exact", variant=None):
    """the id every rank merges for row x (fp32 values representable in dt) split at bounds"""
    x = np.asarray(x, np.float32)
    n = x.shape[0]
    P = len(bounds) - 1
    sh = [(bounds[q], bounds[q + 1]) for q in range(P)]
    key = keys_of(x, dt)
    ids = np.arange(n)
    # phase 0: the shards' argmaxes (NaN first, the lower id on ties); phase 1 merges them in rank order
    rec0 = []
    for a, e in sh:
        xs = x[a:e]
        i = int(np.argmax(xs)) if not np.isnan(xs).any() else int(np.flatnonzero(np.isnan(xs))[0])
        rec0.append((xs[i], a + i))
    m, gid = rec0[0]
    for v, i in rec0[1:]:
        if bool(S.G.beats(np.float32(v), i, np.float32(m), gid)):
            m, gid = v, i
    greedy, c, kk, p24 = S.params(t, k, p, n)
    if not np.isfinite(m) or greedy:
        return int(gid)
    # phase 1: each shard's level-1 histogram at the row's m and c (the shard's own maximum: shard_max)
    W = np.zeros(n, np.int64)
    for a, e in sh:
        W[a:e] = S.weights(x[a:e], x[a:e].max() if variant == "shard_max" else m, c, form)
    hb = key >> 8
    rec1 = []
    for a, e in sh:
        ms = np.zeros(256, np.int64)
        np.add.at(ms, hb[a:e], W[a:e])
        rec1.append((np.bincount(hb[a:e], minlength=256), ms))
    cnt1 = sum(r[0] for r in rec1)
    mass1 = [sum(int(r[1][b]) for r in rec1) for b in range(256)]
    _, first = np.unique(key, return_index=True)  # the weight of a key: the same for all its elements (up to shard_max)
    wkey = {int(key[i]): int(W[i]) for i in first}

    def level2(h):  # each rank's counts of the low byte within high byte h
        return [np.bincount(key[a:e][hb[a:e] == h] & 255, minlength=256) for a, e in sh]

    def finish(h, T, ac1, am1, by_mass, recs):  # the key K and rank j of a selection begun at high byte h
        tot2 = sum(recs)
        m2 = [int(tot2[b]) * wkey.get((h << 8) | b, 0) for b in range(256)]
        lo, ac, am = scan(tot2, m2, by_mass, T - (am1 if by_mass else ac1))
        K = (h << 8) | lo
        ac, am, w = ac + ac1, am + am1, wkey.get(K, 0)
        j = T - ac if not by_mass else ((T - am + w - 1) // w if w else 1)
        return K, j, am + j * w

    # phases 2, 3: top-k; S_k
    if kk == n:
        Sk = sum(mass1)
    elif variant == "topk_per_shard":  # every shard keeps its own first k
        Sk = 0
        for a, e in sh:
            o = a + np.lexsort((ids[a:e], -key[a:e]))
            Sk += int(W[o[:kk]].sum())
    else:
        h, ac1, am1 = scan(cnt1, mass1, False, kk)
        _, _, Sk = finish(h, kk, ac1, am1, False, level2(h))
    # phases 3, 4: top-p; S_p
    Sp = Sk
    if p24 < S.P24:
        Pt = max(1, (p24 * Sk + S.P24 - 1) >> 24)
        h, ac1, am1 = scan(cnt1, mass1, True, Pt)
        _, _, Sp = finish(h, Pt, ac1, am1, True, level2(h))
    if variant == "u_rank_sp":  # U from rank 0's share of the nucleus weight
        o = np.lexsort((ids, -key))
        cum = np.cumsum(W[o])
        npl = int(np.searchsorted(cum, Sp, side="left")) + 1
        nuc = o[:npl]
        Sp = int(W[nuc[nuc < bounds[1]]].sum())
    U = (int(S.draw_u24(seed, off)) * Sp) >> 24
    # phases 4, 5: the draw's key K and its rank j; the ranks' counts of K are their phase-4 records at K's low byte
    h, ac1, am1 = scan(cnt1, mass1, True, U + 1)
    rec4 = level2(h)
    K, j, _ = finish(h, U + 1, ac1, am1, True, rec4)
    cnt = [int(r[K & 255]) for r in rec4]
    rec5 = []
    for q, (a, e) in enumerate(sh):
        pre = sum(cnt[q + 1:]) if variant == "tie_high_rank" else sum(cnt[:q])
        if pre < j <= pre + cnt[q]:
            jl = min(j, cnt[q]) if variant == "no_prefix" else j - pre
            e_loc = int(np.flatnonzero(key[a:e] == K)[jl - 1])
            rec5.append(e_loc if variant == "drop_offset" else a + e_loc)
        else:
            rec5.append(-1)
    held = [v for v in rec5 if v >= 0]
    assert len(held) == 1, rec5
    return held[0]
