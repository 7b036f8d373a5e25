"""Qwen3-8B decode on one GPU: int4 per-channel weights, bf16 KV, ctx 2048 (the bench.py workload on Qwen3 shapes).

  * tokens/s of CUDA-graph-replayed steps at batch 64, 8 and 1 (one set of weights and caches, DecodeStack.set_batch), and
    per-kernel µs at each batch (bench.kernel_rooflines: CUDA events over graph-replayed launches, one layer per launch);
  * the cost of the per-head Q/K RMSNorm inside the step: the same stack, weights and caches stepped with the norm switched
    off (cfg.qk_norm = False, a graph of its own), the two graphs alternated in `--rounds` rounds; medians reported;
  * the span-cache append alone at Qwen3-8B shapes (B = 64: 32 q + 8 k + 8 v head rows per token), with and without the
    fused norm, alternated the same way (µs per launch, each launch on another layer's cache);
  * the card's name and power limit, read in the same run.
Prints one JSON line.  Usage (the DESIGN.md §5 Qwen3 table): python tools/qwen3_bench.py --steps 30 --warmup 5
"""
import argparse
import dataclasses
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "dash-infer_b200", "python"))

import torch  # noqa: E402

import bench  # noqa: E402
from b200spark import model, ops  # noqa: E402


def capture(st, qk_norm):
    st.cfg = dataclasses.replace(st.cfg, qk_norm=qk_norm)
    st.graph = None
    st.capture()
    return st.graph, st.launches_per_step


def step_ms(st, graph, ctx, K, W):
    st.graph = graph
    bench.rewind(st, ctx)
    ms, _ = bench.timed_steps(st, K, W, torch, None, 1)
    return ms / K


def append_us(st, qk_norm, rounds):
    fns = [(lambda L=L: ops._cache_append(L["cache"], st.qkv, st.lens_old, q_out=st.q, rope=st.rope,
                                          qk_norm=(L["qn"], L["kn"], st.cfg.eps) if qk_norm else None)) for L in st.layers]
    return bench.time_kernel_loop(fns, rounds, torch) * 1e6


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=20).stdout.strip()
        name, power = [x.strip() for x in r.split(",")]
        return name, power
    except Exception:
        return torch.cuda.get_device_name(0), None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--ctx", type=int, default=2048)
    ap.add_argument("--batches", default="64,8,1")
    ap.add_argument("--rounds", type=int, default=5, help="alternations of the with / without-norm measurements")
    ap.add_argument("--layers", type=int, default=None, help="debug: fewer layers (not a Qwen3-8B number)")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "qwen3_bench measures on the GPU; there is no CPU fallback"
    name, power = gpu_info()
    batches = [int(b) for b in args.batches.split(",")]
    K, W, ctx = args.steps, max(args.warmup, 3), args.ctx
    cfg = model.QWEN3_8B
    st = model.DecodeStack(cfg, max(batches), ctx + W + K + 16, wbits=4, group=-1, kv="none", span=128, layers=args.layers)
    st.set_context(ctx)
    hbm_peak, _ = bench.peaks()
    out = {"model": cfg.name + ("" if args.layers is None else " (%d layers: debug)" % args.layers), "wbits": 4, "group": -1,
           "kv": "bf16", "ctx": ctx, "steps": K, "rounds": args.rounds, "gpu": name, "power_limit": power, "batches": {}}
    for B in batches:
        st.set_batch(B)
        st.ids.copy_(torch.randint(0, cfg.vocab, (B,), generator=torch.Generator().manual_seed(4321)).cuda())
        g_on, n_on = capture(st, True)
        g_off, n_off = capture(st, False)
        on, off = [], []
        for _ in range(args.rounds):
            on.append(step_ms(st, g_on, ctx, K, W))
            off.append(step_ms(st, g_off, ctx, K, W))
        ms_on, ms_off = statistics.median(on), statistics.median(off)
        st.cfg = dataclasses.replace(st.cfg, qk_norm=True)
        st.graph = g_on
        rec = {"tokens_per_s": round(B * 1e3 / ms_on, 1), "ms_per_step": round(ms_on, 4),
               "no_norm_tokens_per_s": round(B * 1e3 / ms_off, 1), "no_norm_ms_per_step": round(ms_off, 4),
               "norm_cost_pct": round(100 * (ms_on - ms_off) / ms_off, 2),
               "ms_per_step_all": [round(v, 4) for v in on], "no_norm_ms_per_step_all": [round(v, 4) for v in off],
               "launches_per_step": n_on, "no_norm_launches_per_step": n_off,
               "kernels": {k: v["us"] for k, v in bench.kernel_rooflines(st, cfg, hbm_peak, torch).items()}}
        if B == max(batches):
            bench.rewind(st, ctx)
            a_on, a_off = [], []
            for _ in range(args.rounds):
                a_on.append(append_us(st, True, 4))
                a_off.append(append_us(st, False, 4))
            rec["kernels"]["cache_append[B=%d, 48 head rows, qk_norm]" % B] = round(statistics.median(a_on), 2)
            rec["kernels"]["cache_append[B=%d, 48 head rows]" % B] = round(statistics.median(a_off), 2)
            rec["append_us_all"] = {"qk_norm": [round(v, 2) for v in a_on], "plain": [round(v, 2) for v in a_off]}
        out["batches"][str(B)] = rec
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
