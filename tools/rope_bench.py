"""Cost of the scaled rotary (a YaRN frequency table read by the span-cache append) on one GPU.

  * the span-cache append alone at Qwen2-7B heads (28 q + 4 k + 4 v head rows per token) at batch 1 and 64, with the
    frequencies computed (base^(-2f/128)) and read from a YaRN table, alternated in `--rounds` rounds (µs per launch, each
    launch on another layer's cache; medians);
  * the Qwen2.5-7B decode step (int4 per-channel, bf16 KV, ctx 2048) at batch 1, 8 and 64 with rope_scaling on (the
    YaRN x4 table, built once and held while its graph is replayed) and off (the same stack, weights and caches, a graph of
    its own), alternated; medians, per-round range, launches per step; after the timing each graph's step is checked bit
    for bit against an eager step from the same state;
  * one batch-1 step at ctx 65536 (past Qwen2.5's native 32768) with the table;
  * the card's name and power limit, read in the same run.
Prints one JSON line.  Usage (the DESIGN.md §3.3 table): python tools/rope_bench.py --steps 30 --warmup 5
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


def set_scaling(st, table, on):
    """switch the stack between the YaRN table and the computed base frequencies (same weights and caches).  table: the
    stack's (inv_freq, attn_factor), built once by the caller and held for the whole run, because a captured graph keeps
    only the table's address, not a reference to it."""
    st.cfg = dataclasses.replace(st.cfg, rope_scaling=model.YARN_4X_32K if on else None)
    st.rope = table if on else (st.cfg.rope_base, st.head)


def capture(st, table, on):
    set_scaling(st, table, on)
    st.graph = None
    st.capture()
    return st.graph, st.launches_per_step


def replay_matches_eager(st, graph, ctx):
    """the captured step's logits equal an eager step's from the same state, bit for bit (the graph reads live inputs)"""
    ids = (torch.arange(st.ids.numel(), device="cuda", dtype=torch.int64) * 97 + 11) % st.cfg.vocab
    out = []
    for g in (graph, None):
        st.graph = g
        bench.rewind(st, ctx)
        st.ids.copy_(ids)
        st.step()
        torch.cuda.synchronize()
        out.append(st.logits.clone())
    st.graph = graph
    return torch.equal(out[0], out[1])


def step_ms(st, graph, ctx, K, W):
    st.graph = graph
    bench.rewind(st, ctx)
    ms, _ = bench.timed_steps(st, K, W, torch, None, 1)
    return ms / K


def append_us(st, table, on, rounds):
    set_scaling(st, table, on)
    fns = [(lambda L=L: ops._cache_append(L["cache"], st.qkv, st.lens_old, q_out=st.q, rope=st.rope)) for L in st.layers]
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
    ap.add_argument("--long-ctx", type=int, default=65536)
    ap.add_argument("--batches", default="1,8,64")
    ap.add_argument("--rounds", type=int, default=5, help="alternations of the scaled / unscaled measurements")
    ap.add_argument("--layers", type=int, default=None, help="debug: fewer layers (not a Qwen2.5-7B number)")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "rope_bench measures on the GPU; there is no CPU fallback"
    name, power = gpu_info()
    batches = [int(b) for b in args.batches.split(",")]
    K, W, ctx = args.steps, max(args.warmup, 3), args.ctx
    cfg = model.QWEN25_7B
    out = {"model": cfg.name + ("" if args.layers is None else " (%d layers: debug)" % args.layers), "rope_scaling": cfg.rope_scaling,
           "wbits": 4, "group": -1, "kv": "bf16", "ctx": ctx, "steps": K, "rounds": args.rounds, "gpu": name,
           "power_limit": power, "append_us": {}, "batches": {}}
    st = model.DecodeStack(cfg, max(batches), ctx + W + K + 16, wbits=4, group=-1, kv="none", span=128, layers=args.layers)
    st.set_context(ctx)
    table = st.rope  # the YaRN table DecodeStack built on the device; alive until the end of main()
    for B in sorted({1, 64} & set(batches) or {max(batches)}):
        st.set_batch(B)
        bench.rewind(st, ctx)
        a_on, a_off = [], []
        for _ in range(args.rounds):
            a_on.append(append_us(st, table, True, 4))
            a_off.append(append_us(st, table, False, 4))
        out["append_us"][str(B)] = {"table": round(statistics.median(a_on), 3), "base": round(statistics.median(a_off), 3),
                                    "table_all": [round(v, 3) for v in a_on], "base_all": [round(v, 3) for v in a_off]}
    for B in batches:
        st.set_batch(B)
        st.ids.copy_(torch.randint(0, cfg.vocab, (B,), generator=torch.Generator().manual_seed(4321)).cuda())
        g_on, n_on = capture(st, table, True)
        g_off, n_off = capture(st, table, False)
        on, off = [], []
        for _ in range(args.rounds):
            on.append(step_ms(st, g_on, ctx, K, W))
            off.append(step_ms(st, g_off, ctx, K, W))
        # both graphs still compute what their eager steps compute (the scaled one with the table, read after the timing)
        set_scaling(st, table, True)
        ok_on = replay_matches_eager(st, g_on, ctx)
        set_scaling(st, table, False)
        ok_off = replay_matches_eager(st, g_off, ctx)
        assert ok_on and ok_off, (B, ok_on, ok_off)
        ms_on, ms_off = statistics.median(on), statistics.median(off)
        out["batches"][str(B)] = {
            "tokens_per_s": round(B * 1e3 / ms_on, 1), "ms_per_step": round(ms_on, 4),
            "unscaled_tokens_per_s": round(B * 1e3 / ms_off, 1), "unscaled_ms_per_step": round(ms_off, 4),
            "scaling_cost_pct": round(100 * (ms_on - ms_off) / ms_off, 2),
            "ms_per_step_range": [round(min(on), 4), round(max(on), 4)],
            "unscaled_ms_per_step_range": [round(min(off), 4), round(max(off), 4)],
            "ms_per_step_all": [round(v, 4) for v in on], "unscaled_ms_per_step_all": [round(v, 4) for v in off],
            "launches_per_step": n_on, "unscaled_launches_per_step": n_off, "replay_matches_eager": True}
    del st, g_on, g_off, table
    torch.cuda.empty_cache()
    if args.long_ctx:
        L = args.long_ctx
        st = model.DecodeStack(cfg, 1, L + W + K + 16, wbits=4, group=-1, kv="none", span=128, layers=args.layers)
        st.set_context(L)
        st.ids.copy_(torch.tensor([1234], device="cuda"))
        st.capture()
        ms = step_ms(st, st.graph, L, K, W)
        out["long_ctx"] = {"ctx": L, "batch": 1, "tokens_per_s": round(1e3 / ms, 1), "ms_per_step": round(ms, 4),
                           "launches_per_step": st.launches_per_step}
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
