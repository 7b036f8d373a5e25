"""GLM-4-9B decode on one GPU: int4 per-channel weights, ctx 2048 (the bench.py workload on GLM-4 shapes).

  * tokens/s of CUDA-graph-replayed steps at batch 64, 8 and 1 (one set of weights and caches, DecodeStack.set_batch), with
    a bf16 and an int8 KV cache, and per-kernel µs at each batch (bench.kernel_rooflines);
  * the span-cache append alone at GLM-4-9B shapes (B = 64: 32 q + 2 k + 2 v head rows per token) with the interleaved
    rotary GLM runs and with the NeoX pairing over the same 64 dims, alternated in `--rounds` rounds (µs per launch, each
    launch on another layer's cache); medians reported;
  * the card's name and power limit, read in the same run.
Prints one JSON line.  Usage (the DESIGN.md §5 GLM table): python tools/glm_bench.py --steps 30 --warmup 5
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "dash-infer_b200", "python"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch  # noqa: E402

import bench  # noqa: E402
from b200spark import model, ops  # noqa: E402
from qwen3_bench import gpu_info, step_ms  # noqa: E402


def append_us(st, rope, rounds):
    fns = [(lambda L=L: ops._cache_append(L["cache"], st.qkv, st.lens_old, q_out=st.q, rope=rope)) for L in st.layers]
    return bench.time_kernel_loop(fns, rounds, torch) * 1e6


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--ctx", type=int, default=2048)
    ap.add_argument("--batches", default="64,8,1")
    ap.add_argument("--kv", default="bf16,i8")
    ap.add_argument("--rounds", type=int, default=5, help="alternations of the interleaved / NeoX append measurements")
    ap.add_argument("--layers", type=int, default=None, help="debug: fewer layers (not a GLM-4-9B number)")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "glm_bench measures on the GPU; there is no CPU fallback"
    name, power = gpu_info()
    batches = [int(b) for b in args.batches.split(",")]
    K, W, ctx = args.steps, max(args.warmup, 3), args.ctx
    cfg = model.GLM4_9B
    hbm_peak, _ = bench.peaks()
    out = {"model": cfg.name + ("" if args.layers is None else " (%d layers: debug)" % args.layers), "wbits": 4, "group": -1,
           "ctx": ctx, "steps": K, "rounds": args.rounds, "gpu": name, "power_limit": power, "kv": {}}
    for kv in args.kv.split(","):
        st = model.DecodeStack(cfg, max(batches), ctx + W + K + 16, wbits=4, group=-1, kv=kv, span=128, layers=args.layers)
        st.set_context(ctx)
        recs = {}
        for B in batches:
            st.set_batch(B)
            st.ids.copy_(torch.randint(0, cfg.vocab, (B,), generator=torch.Generator().manual_seed(4321)).cuda())
            st.graph = None
            st.capture()
            ms = [step_ms(st, st.graph, ctx, K, W) for _ in range(3)]
            m = statistics.median(ms)
            rec = {"tokens_per_s": round(B * 1e3 / m, 1), "ms_per_step": round(m, 4), "ms_per_step_all": [round(v, 4) for v in ms],
                   "launches_per_step": st.launches_per_step,
                   "kernels": {k: v["us"] for k, v in bench.kernel_rooflines(st, cfg, hbm_peak, torch).items()}}
            if B == max(batches):
                bench.rewind(st, ctx)
                il, neox = st.rope, (cfg.rope_base, cfg.rotary_dim)
                a_il, a_neox = [], []
                for _ in range(args.rounds):
                    a_il.append(append_us(st, il, 4))
                    a_neox.append(append_us(st, neox, 4))
                rows = cfg.n_heads + 2 * cfg.n_kv
                rec["kernels"]["cache_append[B=%d, %d head rows, interleaved]" % (B, rows)] = round(statistics.median(a_il), 2)
                rec["kernels"]["cache_append[B=%d, %d head rows, neox]" % (B, rows)] = round(statistics.median(a_neox), 2)
                rec["append_us_all"] = {"interleaved": [round(v, 2) for v in a_il], "neox": [round(v, 2) for v in a_neox]}
            recs[str(B)] = rec
        out["kv"][kv] = recs
        del st
        torch.cuda.empty_cache()
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
