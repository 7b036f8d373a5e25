"""Multi-token verify steps (speculative decoding) on one GPU: Qwen2-7B int4 (per-channel), bf16 KV, ctx 2048.

For each q_len T in {1, 2, 4, 8} and batch 1 and 8: ms per CUDA-graph-replayed decode step (T = 1: the ordinary step) and
the attention kernel's µs (layer 0, eager launches).  Two draft sets bound what any drafter can get:
  * "own": the model's own greedy continuation (found by repeating the step until its drafts equal its predictions), so
    every sequence accepts all T;
  * "random": uniformly drawn drafts, so (almost surely) every sequence accepts 1.
Each timed replay verifies the same step: after it, the lengths and column 0 of the token array are restored (three small
copies, inside the timed loop).  tokens/s = the accepted tokens the accept kernel reported / the step time.
Prints one JSON line.

Usage (the DESIGN.md §5 table): python tools/spec_bench.py --steps 30 --warmup 5

--tree: draft trees (DecodeStack(tree=True)) against chains of the same size, for T in {4, 8, 16} nodes and batch 1 and 8:
  * ms per CUDA-graph-replayed step of a tree step and of the chain step (the same stack's weights and caches), and the
    accepted tokens/s for two draft sets: "own", a tree whose LAST branch (nodes T/2 .. T-1, hanging off the root) holds the
    model's greedy continuation behind a first branch of random drafts, so T/2 + 1 tokens are accepted and compaction moves
    T/2 rows per layer; "random", random parents and drafts (almost surely 1 accepted).  The chain's "own" accepts all T;
  * the attention kernel's µs for run_tree (the random tree) and run_tokens (layer 0, eager launches);
  * the µs of spec_accept_tree + cache_compact (28 layers): a CUDA graph of both plus the state restore, minus a graph of
    the restore alone.
Replaying the same tree step stays valid after compaction: the step rewrites all T slots past the restored length before
anything reads them, and compaction only writes inside those slots.
Usage (the DESIGN.md §5 tree table): python tools/spec_bench.py --tree --steps 30 --warmup 5

--sample: sampled verification (DecodeStack(sampled_verify=True)) against greedy verification on the same stack, for T in
{4, 8, 16}, batch 1 and 8, chains and trees, at t = 0.7, k = 50, p = 0.9:
  * ms per CUDA-graph-replayed step of each, alternated over --rounds rounds: medians and the spread (min, max);
  * µs per launch of b2_sample_tokens and of b2_argmax on [B*T, 152064] bf16 rows (a graph of 20 launches);
  * accepted tokens/s of the sampled step for two draft sets: "own", the continuation a single-token sampled stack
    (sample=True, same weights, caches, seeds and offsets) draws, on a chain, or on a tree's last branch behind a first
    branch of random drafts; "random", random drafts (and random parents).  "own" is not accepted whole: verify rows pass
    the GEMMs at M = B*T, so their logits differ from the single-token step's by rounding, and a draw can change.
Usage (the DESIGN.md §5 sampled-verification table): python tools/spec_bench.py --sample --steps 30 --warmup 5

--ngram: the on-device n-gram drafter (DecodeStack(ngram=(1, 4, width))):
  * µs per launch of b2_ngram_draft (a graph of 20) at T = 8, B = 1 / 8 / 64, history L = 2K / 32K / 128K, width 1 (chain)
    and 4 (tree), over random histories (the full scan) and periodic ones (the candidate walk stops early); and of
    b2_history_append_tokens (8 tokens per sequence);
  * ms per CUDA-graph-replayed verify step with the drafter against the same step with host-written drafts (the drafter's
    own, so both verify the same tokens), alternated over --rounds rounds: medians and the spread; T = 4 / 8 / 16, B = 1
    and 8, chain and tree;
  * generation at T = 8: --steps graph replays back to back with nothing restored, from prompts that repeat a random
    61-token segment and from random prompts: accepted tokens per step and tokens/s, against the q_len = 1 step on the
    same weights.  The weights are synthetic, so the acceptance says nothing about a real model's.
Usage (the DESIGN.md §5 drafter table): python tools/spec_bench.py --ngram --steps 30 --warmup 5
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "dash-infer_b200", "python"))

import torch  # noqa: E402

from b200spark import model  # noqa: E402


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=20).stdout.strip()
        name, power = [x.strip() for x in out.split(",")]
        return name, power
    except Exception:
        return torch.cuda.get_device_name(0), None


def time_ms(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def graph_of(fn):
    fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    torch.cuda.synchronize()
    return g


def tree_main(args, name, power):
    from b200spark import ops
    cfg = model.QWEN2_7B
    res = []
    gen = torch.Generator(device="cuda").manual_seed(6)
    for T in (4, 8, 16):
        st = model.DecodeStack(cfg, 8, args.ctx + 64, wbits=4, group=-1, kv="none", span=128, q_len=T, tree=True)
        st.set_context(args.ctx)
        h = T // 2
        own_tree = [0] + [0 if t in (1, h) else t - 1 for t in range(1, T)]  # nodes 1 .. h-1 and h .. T-1: two branches
        for B in (8, 1):
            st.set_batch(B)
            lo, ln = st.lens_old.clone(), st.lens_new.clone()
            st.tokens.copy_(torch.randint(0, cfg.vocab, st.tokens.shape, generator=gen, device="cuda"))
            row = {"batch": B, "q_len": T}
            # the chain op sequence of the same stack: b2_spec_accept, no compaction
            st.tree = False
            st.capture()
            tk = st.tokens.clone()
            for _ in range(T):  # the model's greedy continuation as a chain: each pass fixes at least one more draft
                st.step()
                tk[:, 1:] = st.pred[:, :-1]
                st.tokens.copy_(tk)
                st.lens_old.copy_(lo); st.lens_new.copy_(ln)
            greedy = tk[:, 1:].clone()
            sets = {"chain_own": (None, tk.clone()),
                    "chain_random": (None, torch.cat([tk[:, :1], torch.randint(0, cfg.vocab, (B, T - 1), generator=gen,
                                                                                device="cuda")], 1))}
            own = tk.clone()
            own[:, 1:h] = torch.randint(0, cfg.vocab, (B, h - 1), generator=gen, device="cuda")
            own[:, h:] = greedy[:, :T - h]
            cpu_gen = torch.Generator().manual_seed(7 + T + B)
            rnd_par = torch.tensor([[0] + [int(torch.randint(0, t, (1,), generator=cpu_gen).item()) for t in range(1, T)]
                                    for _ in range(B)], dtype=torch.int32)
            sets["tree_own"] = (torch.tensor([own_tree] * B, dtype=torch.int32), own)
            sets["tree_random"] = (rnd_par, sets["chain_random"][1].clone())
            for key, (par, tokens) in sets.items():
                if (par is not None) != st.tree:
                    st.tree = par is not None
                    if st.tree:
                        st.parents.copy_(par)
                    st.capture()
                if par is not None:
                    st.parents.copy_(par)
                st.tokens.copy_(tokens)

                def step():
                    st.step()
                    st.lens_old.copy_(lo); st.lens_new.copy_(ln)
                    st.tokens.copy_(tokens)

                ms = time_ms(step, args.steps, args.warmup)
                acc = int(st.accepted.sum().item())
                row["ms_" + key] = round(ms, 4)
                row["accepted_" + key] = acc
                row["tok_s_" + key] = round(acc / ms * 1e3, 1)
            L = st.layers[0]
            st.parents.copy_(rnd_par)
            row["attn_us_tree"] = round(1e3 * time_ms(
                lambda: st.attn.run_tree(st.q, L["cache"], st.lens_new, st.parents, T, st.max_len, st.ws, out=st.ao), 200, 20), 2)
            row["attn_us_chain"] = round(1e3 * time_ms(
                lambda: st.attn.run_tokens(st.q, L["cache"], st.lens_new, T, st.max_len, st.ws, out=st.ao), 200, 20), 2)
            # accept + compaction on the "own" tree (paths of T/2 + 1 nodes): graph with the restore minus the restore alone
            st.parents.copy_(sets["tree_own"][0])
            caches = [x["cache"] for x in st.layers]
            tokens = sets["tree_own"][1]

            def restore():
                st.lens_old.copy_(lo); st.lens_new.copy_(ln)
                st.tokens.copy_(tokens)

            def accept_compact():
                restore()
                ops.spec_accept_tree(st.accepted, st.path, st.next_ids, st.lens_old, st.lens_new, st.tokens, st.pred, st.parents)
                ops.cache_compact(caches, st.lens_old, st.accepted, st.path, T)

            g1, g0 = graph_of(accept_compact), graph_of(restore)
            reps = 50
            t1 = time_ms(lambda: [g1.replay() for _ in range(reps)], 10, 3)
            t0 = time_ms(lambda: [g0.replay() for _ in range(reps)], 10, 3)
            row["accept_compact_us"] = round(1e3 * (t1 - t0) / reps, 2)
            restore()
            res.append(row)
            print(json.dumps(row), file=sys.stderr, flush=True)
        del st
        torch.cuda.empty_cache()
    print(json.dumps({"gpu": name, "power_limit": power, "model": "Qwen2-7B int4 per-channel, bf16 KV", "ctx": args.ctx,
                      "tree": True, "results": res}))


def sample_main(args, name, power):
    from b200spark import ops
    cfg = model.QWEN2_7B
    t, k, p = 0.7, 50, 0.9
    gen = torch.Generator(device="cuda").manual_seed(8)
    seeds, offs = torch.arange(8, dtype=torch.int64, device="cuda") * 7919 + 1, torch.full((8,), 1000, dtype=torch.int64,
                                                                                          device="cuda")
    one = model.DecodeStack(cfg, 8, args.ctx + 64, wbits=4, group=-1, kv="none", span=128, sample=True)
    one.set_context(args.ctx)
    one.set_sampling(temperature=t, top_k=k, top_p=p, seeds=seeds, offsets=offs)
    first = torch.randint(0, cfg.vocab, (8,), generator=gen, device="cuda")

    def continuation(B, n):
        """the single-token sampled stack's next n tokens after `first`, from the context and offsets of the verify step"""
        one.set_batch(B)
        one.lens_old.fill_(args.ctx); one.lens_new.fill_(args.ctx + 1)
        one.offsets.copy_(offs[:B]); one.ids.copy_(first[:B])
        out = []
        for _ in range(n):
            out.append(one.step().clone())
            one.ids.copy_(out[-1])
        return torch.stack(out, 1)

    res = []
    for T in (4, 8, 16):
        st = model.DecodeStack(cfg, 8, args.ctx + 64, wbits=4, group=-1, kv="none", span=128, q_len=T, tree=True,
                               sampled_verify=True)
        st.set_context(args.ctx)
        h = T // 2
        own_tree = [0] + [0 if u in (1, h) else u - 1 for u in range(1, T)]  # nodes 1 .. h-1 and h .. T-1: two branches
        for B in (8, 1):
            st.set_batch(B)
            st.set_sampling(temperature=t, top_k=k, top_p=p, seeds=seeds[:B], offsets=offs[:B])
            lo, ln, off0 = st.lens_old.clone(), st.lens_new.clone(), st.offsets.clone()
            cont = continuation(B, T)
            lg = (torch.randn(B * T, cfg.vocab, generator=gen, device="cuda") * 3).to(torch.bfloat16)
            ids = torch.empty(B * T, dtype=torch.int64, device="cuda")
            cpu_gen = torch.Generator().manual_seed(7 + T + B)
            par_rnd = torch.tensor([[0] + [int(torch.randint(0, u, (1,), generator=cpu_gen).item()) for u in range(1, T)]
                                    for _ in range(B)], dtype=torch.int32, device="cuda")
            launches = {"argmax": lambda: ops.argmax(lg, out=ids),
                        "sample_tokens": lambda: ops.sample_tokens(lg, T, st.temperature, st.top_k, st.top_p, st.seeds, st.offsets,
                                                                   parents=par_rnd, out=ids)}
            for form in ("chain", "tree"):
                st.tree = form == "tree"
                rnd = torch.cat([first[:B, None], torch.randint(0, cfg.vocab, (B, T - 1), generator=gen, device="cuda")], 1)
                own = rnd.clone()
                if st.tree:
                    own[:, h:] = cont[:, :T - h]
                else:
                    own[:, 1:] = cont[:, :T - 1]
                row = {"batch": B, "q_len": T, "form": form}
                graphs = {}
                for mode in ("greedy", "sampled"):
                    st.sv = mode == "sampled"
                    if st.tree:
                        st.parents.copy_(torch.tensor([own_tree] * B, dtype=torch.int32))
                    st.tokens.copy_(own)
                    graphs[mode] = st.capture()
                for drafts, (tokens, par) in {"own": (own, own_tree), "random": (rnd, None)}.items():
                    if st.tree:
                        st.parents.copy_(par_rnd if par is None else torch.tensor([par] * B, dtype=torch.int32))

                    def step():
                        st.graph.replay()
                        st.lens_old.copy_(lo); st.lens_new.copy_(ln)
                        st.tokens.copy_(tokens); st.offsets.copy_(off0)

                    ms = {"greedy": [], "sampled": []}
                    for _ in range(args.rounds):  # alternated
                        for mode in ms:
                            st.graph = graphs[mode]
                            ms[mode].append(time_ms(step, args.steps, args.warmup))
                    st.graph = graphs["sampled"]
                    step()
                    acc = int(st.accepted.sum().item())
                    for mode, v in ms.items():
                        row["ms_%s_%s" % (mode, drafts)] = round(statistics.median(v), 4)
                        row["ms_%s_%s_spread" % (mode, drafts)] = [round(min(v), 4), round(max(v), 4)]
                    row["cost_pct_" + drafts] = round(100 * (statistics.median(ms["sampled"]) / statistics.median(ms["greedy"]) - 1), 2)
                    row["accepted_" + drafts] = acc
                    row["tok_s_" + drafts] = round(acc / statistics.median(ms["sampled"]) * 1e3, 1)
                res.append(row)
                print(json.dumps(row), file=sys.stderr, flush=True)
            us = {}
            for name_, f in launches.items():
                g = graph_of(lambda: [f() for _ in range(20)])
                us[name_] = round(1e3 * time_ms(g.replay, 10, 3) / 20, 2)
            res[-1]["launch_us"] = res[-2]["launch_us"] = us
            st.sv, st.graph = True, None
        del st
        torch.cuda.empty_cache()
    print(json.dumps({"gpu": name, "power_limit": power, "model": "Qwen2-7B int4 per-channel, bf16 KV", "ctx": args.ctx,
                      "sample": {"temperature": t, "top_k": k, "top_p": p}, "rounds": args.rounds, "results": res}))


def _fill_history(h, B, L, kind, gen):
    """slots 0 .. B-1 of h := L tokens: "random" ids (the drafter scans everything) or a repeated random segment of 37
    tokens ("periodic": the longest matches are the most recent, so the candidate walk stops in its first chunk)"""
    if kind == "random":
        tok = torch.randint(0, 152064, (B, L), generator=gen, device="cuda", dtype=torch.int32)
    else:
        seg = torch.randint(0, 152064, (B, 37), generator=gen, device="cuda", dtype=torch.int32)
        tok = seg.repeat(1, L // 37 + 1)[:, :L]
    h.tokens[:B, :L] = tok
    h.len[:B] = L


def ngram_main(args, name, power):
    from b200spark import ops
    cfg = model.QWEN2_7B
    gen = torch.Generator(device="cuda").manual_seed(9)
    res = {"kernel": [], "step": [], "generate": []}
    # 1. the two launches alone: a graph of 20, µs per launch
    T = 8
    hist = ops.TokenHistory(64, 131072 + 4096, cfg.vocab)
    for kind in ("random", "periodic"):
        for L in (2048, 32768, 131072):
            for B in (1, 8, 64):
                _fill_history(hist, B, L, kind, gen)
                h = hist.view(B)
                tokens = torch.zeros(B, T, dtype=torch.int64, device="cuda")
                tokens[:, 0] = h.tokens[:, L - 1]
                parents = torch.zeros(B, T, dtype=torch.int32, device="cuda")
                row = {"kind": kind, "L": L, "batch": B, "q_len": T}
                for width in (1, 4):
                    par = parents if width > 1 else None
                    g = graph_of(lambda: [ops.ngram_draft(h, tokens, par, 1, 4, width) for _ in range(20)])
                    row["draft_us_w%d" % width] = round(1e3 * time_ms(g.replay, 10, 3) / 20, 2)
                if kind == "random" and L == 2048:  # T accepted tokens per sequence and launch
                    acc = torch.full((B,), T, dtype=torch.int32, device="cuda")
                    pred = torch.randint(0, cfg.vocab, (B, T), generator=gen, device="cuda")
                    g = graph_of(lambda: [h.append_tokens(pred, acc) for _ in range(20)])
                    row["append_us"] = round(1e3 * time_ms(g.replay, 10, 3) / 20, 2)
                res["kernel"].append(row)
                print(json.dumps(row), file=sys.stderr, flush=True)
    del hist
    # 2. the verify step with the drafter against the same step with host-written drafts (the drafter's own, so both
    # verify the same tokens), alternated; 3. generation: steps replayed back to back, nothing restored
    seg = torch.randint(0, cfg.vocab, (8, 61), generator=gen, device="cuda").cpu()
    prompts = {"repeat": seg.repeat(1, args.ctx // 61 + 1)[:, :args.ctx],
               "random": torch.randint(0, cfg.vocab, (8, args.ctx), generator=gen, device="cuda").cpu()}
    n_gen = args.steps
    one = None
    for T in (4, 8, 16):
        st = model.DecodeStack(cfg, 8, args.ctx + 16 * n_gen + 64, wbits=4, group=-1, kv="none", span=128, q_len=T, tree=True,
                               ngram=(1, 4, 1))
        st.set_context(args.ctx)
        for B in (8, 1):
            st.set_batch(B)
            for b in range(B):
                st.set_history(b, prompts["repeat"][b])
            lo, ln, hl = st.lens_old.clone(), st.lens_new.clone(), st.history.len.clone()
            tk0 = st.tokens.clone()
            for form, ngram in (("chain", (1, 4, 1)), ("tree", (1, 4, min(4, T - 1)))):
                st.tree, st.ngram = form == "tree", ngram
                graphs = {"ngram": st.capture()}
                st.step()  # the drafter's drafts become the host drafts
                torch.cuda.synchronize()
                drafted = (st.tokens.clone(), st.parents.clone())
                st.lens_old.copy_(lo); st.lens_new.copy_(ln); st.history.len.copy_(hl); st.tokens.copy_(tk0)
                st.ngram = None
                st.tokens[:, 1:] = drafted[0][:, 1:]
                st.parents.copy_(drafted[1])
                graphs["host"] = st.capture()
                st.ngram = ngram
                tokens = {"ngram": tk0.clone(), "host": st.tokens.clone()}
                ms = {"ngram": [], "host": []}
                for _ in range(args.rounds):
                    for mode in ms:
                        st.graph = graphs[mode]

                        def step():
                            st.graph.replay()
                            st.lens_old.copy_(lo); st.lens_new.copy_(ln); st.history.len.copy_(hl)
                            st.tokens.copy_(tokens[mode])
                            st.parents.copy_(drafted[1])

                        ms[mode].append(time_ms(step, args.steps, args.warmup))
                row = {"batch": B, "q_len": T, "form": form, "width": ngram[2], "accepted": int(st.accepted.sum())}
                for mode, v in ms.items():
                    row["ms_" + mode] = round(statistics.median(v), 4)
                    row["ms_%s_spread" % mode] = [round(min(v), 4), round(max(v), 4)]
                row["cost_pct"] = round(100 * (statistics.median(ms["ngram"]) / statistics.median(ms["host"]) - 1), 2)
                res["step"].append(row)
                print(json.dumps(row), file=sys.stderr, flush=True)
                if T != 8:
                    continue
                st.graph = graphs["ngram"]
                for pk, pr in prompts.items():  # generation from each prompt kind
                    for b in range(B):
                        st.set_history(b, pr[b])
                    st.lens_old.copy_(lo); st.lens_new.copy_(ln)
                    h0 = st.history.len.clone()
                    torch.cuda.synchronize()
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    for _ in range(n_gen):
                        st.graph.replay()
                    e1.record()
                    torch.cuda.synchronize()
                    ms_ = e0.elapsed_time(e1)
                    toks = int((st.history.len - h0).sum())
                    g_row = {"batch": B, "q_len": T, "form": form, "width": ngram[2], "prompt": pk, "steps": n_gen,
                             "accepted_per_step": round(toks / (n_gen * B), 3), "tok_s": round(toks / ms_ * 1e3, 1),
                             "ms_per_step": round(ms_ / n_gen, 4)}
                    res["generate"].append(g_row)
                    print(json.dumps(g_row), file=sys.stderr, flush=True)
                st.lens_old.copy_(lo); st.lens_new.copy_(ln)
                for b in range(B):
                    st.set_history(b, prompts["repeat"][b])
                st.tokens.copy_(tk0)
        del st
        torch.cuda.empty_cache()
    # the single-token step on the same weights: tokens/s = B / step time
    one = model.DecodeStack(cfg, 8, args.ctx + 64, wbits=4, group=-1, kv="none", span=128)
    one.set_context(args.ctx)
    q1 = {}
    for B in (8, 1):
        one.set_batch(B)
        lo, ln = one.lens_old.clone(), one.lens_new.clone()
        one.capture()

        def step1():
            one.step()
            one.lens_old.copy_(lo); one.lens_new.copy_(ln)

        ms = time_ms(step1, args.steps, args.warmup)
        q1[str(B)] = {"ms_per_step": round(ms, 4), "tok_s": round(B / ms * 1e3, 1)}
    print(json.dumps({"gpu": name, "power_limit": power, "model": "Qwen2-7B int4 per-channel, bf16 KV", "ctx": args.ctx,
                      "ngram": {"n_min": 1, "n_max": 4}, "rounds": args.rounds, "q_len_1": q1, **res,
                      "note": "synthetic weights: the acceptance says nothing about a real model's"}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--ctx", type=int, default=2048)
    ap.add_argument("--tree", action="store_true", help="draft trees against chains (T = 4, 8, 16)")
    ap.add_argument("--sample", action="store_true", help="sampled against greedy verification (T = 4, 8, 16)")
    ap.add_argument("--ngram", action="store_true", help="the on-device n-gram drafter: kernel times, step cost, generation")
    ap.add_argument("--rounds", type=int, default=5, help="--sample, --ngram: alternations of the two steps measured")
    args = ap.parse_args()
    name, power = gpu_info()
    if args.tree:
        return tree_main(args, name, power)
    if args.sample:
        return sample_main(args, name, power)
    if args.ngram:
        return ngram_main(args, name, power)
    res = []
    gen = torch.Generator(device="cuda").manual_seed(5)
    for T in (1, 2, 4, 8):
        st = model.DecodeStack(model.QWEN2_7B, 8, args.ctx + 64, wbits=4, group=-1, kv="none", span=128, q_len=T)
        st.set_context(args.ctx)
        for B in (8, 1):
            st.set_batch(B)
            lo, ln = st.lens_old.clone(), st.lens_new.clone()
            tokens = st.ids if T == 1 else st.tokens
            tokens.copy_(torch.randint(0, model.QWEN2_7B.vocab, tokens.shape, generator=gen, device="cuda"))
            st.capture()
            row = {"batch": B, "q_len": T}
            for drafts in (("own", "random") if T > 1 else ("own",)):
                if T > 1 and drafts == "own":
                    tk = tokens.clone()
                    for _ in range(T):  # each pass fixes at least one more draft
                        st.step()
                        tk[:, 1:] = st.pred[:, :-1]
                        tokens.copy_(tk)
                        st.lens_old.copy_(lo); st.lens_new.copy_(ln)
                elif T > 1:
                    tokens[:, 1:] = torch.randint(0, model.QWEN2_7B.vocab, (B, T - 1), generator=gen, device="cuda")
                tk = tokens.clone()

                def step():
                    st.step()
                    st.lens_old.copy_(lo); st.lens_new.copy_(ln)
                    tokens.copy_(tk)

                ms = time_ms(step, args.steps, args.warmup)
                acc = B if T == 1 else int(st.accepted.sum().item())
                row["ms_" + drafts] = round(ms, 4)
                row["accepted_" + drafts] = acc
                row["tok_s_" + drafts] = round(acc / ms * 1e3, 1)
            L = st.layers[0]
            if T == 1:
                attn = lambda: st.attn(st.q, L["cache"], st.lens_new, st.max_len, st.ws, out=st.ao)  # noqa: E731
            else:
                attn = lambda: st.attn.run_tokens(st.q, L["cache"], st.lens_new, T, st.max_len, st.ws, out=st.ao)  # noqa: E731
            row["attn_us"] = round(1e3 * time_ms(attn, 200, 20), 2)
            res.append(row)
            print(json.dumps(row), file=sys.stderr, flush=True)
        del st
        torch.cuda.empty_cache()
    print(json.dumps({"gpu": name, "power_limit": power, "model": "Qwen2-7B int4 per-channel, bf16 KV", "ctx": args.ctx,
                      "results": res}))


if __name__ == "__main__":
    main()
