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
"""
import argparse
import json
import os
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--ctx", type=int, default=2048)
    ap.add_argument("--tree", action="store_true", help="draft trees against chains (T = 4, 8, 16)")
    args = ap.parse_args()
    name, power = gpu_info()
    if args.tree:
        return tree_main(args, name, power)
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
