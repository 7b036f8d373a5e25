"""Cost of sampling the decode step's token on one GPU.

  * b2_sample against b2_argmax on [B, 152064] bf16 logits at B = 1, 8, 64: µs per launch, CUDA events over launches replayed
    from a CUDA graph (bench.time_kernel_loop), cycling through 4 logits buffers; settings t = 0 (greedy), t = 1 without a
    filter, k = 50, p = 0.9, and t = 0.7 with k = 50 and p = 0.9;
  * the Qwen2-7B step (bench.py's workload: int4 per-channel, bf16 KV, ctx 2048) with sample=True at t = 0.7, k = 50,
    p = 0.9 against the greedy step at B = 64, 8, 1: one set of weights and caches, a graph of each, alternated in `--rounds`
    rounds; medians reported;
  * the card's name and power limit, read in the same run.
Prints one JSON line.  Usage (the DESIGN.md §3.8 table): python tools/sample_bench.py --steps 30 --warmup 5
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
from logprobs_bench import VOCAB, gpu_info  # noqa: E402

SETTINGS = {"t=0": (0.0, 0, 1.0), "t=1": (1.0, 0, 1.0), "k=50": (1.0, 50, 1.0), "p=0.9": (1.0, 0, 0.9),
            "t=0.7,k=50,p=0.9": (0.7, 50, 0.9)}


def kernels_us(B, rounds):
    g = torch.Generator(device="cuda").manual_seed(B)
    bufs = [(torch.randn(B, VOCAB, generator=g, device="cuda") * 3).to(torch.bfloat16) for _ in range(4)]
    ids = torch.empty(B, dtype=torch.int64, device="cuda")
    seeds = torch.arange(B, dtype=torch.int64, device="cuda")
    offs = torch.zeros(B, dtype=torch.int64, device="cuda")
    fns = {"argmax": [lambda x=x: ops.argmax(x, out=ids) for x in bufs]}
    for name, (t, k, p) in SETTINGS.items():
        prm = (torch.full((B,), t, device="cuda"), torch.full((B,), k, dtype=torch.int32, device="cuda"),
               torch.full((B,), p, device="cuda"))
        fns["sample[%s]" % name] = [lambda x=x, prm=prm: ops.sample(x, *prm, seeds, offs, out=ids) for x in bufs]
    res = {name: [] for name in fns}
    for _ in range(rounds):  # alternated
        for name, f in fns.items():
            res[name].append(bench.time_kernel_loop(f, 25, torch) * 1e6)
    return {name: round(statistics.median(v), 2) for name, v in res.items()}


def step_ms(st, graph, ctx, K, W):
    st.graph = graph
    bench.rewind(st, ctx)
    ms, _ = bench.timed_steps(st, K, W, torch, None, 1)
    return ms / K


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--ctx", type=int, default=2048)
    ap.add_argument("--batches", default="64,8,1")
    ap.add_argument("--rounds", type=int, default=5, help="alternations of the sampled / greedy measurements")
    ap.add_argument("--layers", type=int, default=None, help="debug: fewer layers (not a Qwen2-7B number)")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "sample_bench measures on the GPU; there is no CPU fallback"
    name, power = gpu_info()
    batches = [int(b) for b in args.batches.split(",")]
    K, W, ctx = args.steps, max(args.warmup, 3), args.ctx
    out = {"gpu": name, "power_limit": power, "kernels_us": {}, "model": model.QWEN2_7B.name, "ctx": ctx, "steps": K,
           "rounds": args.rounds, "batches": {}}
    for B in (1, 8, 64):
        out["kernels_us"][str(B)] = kernels_us(B, args.rounds)
    cfg = model.QWEN2_7B
    st = model.DecodeStack(cfg, max(batches), ctx + W + K + 16, wbits=4, group=-1, kv="none", span=128, layers=args.layers,
                           sample=True)
    st.set_context(ctx)
    for B in batches:
        st.set_batch(B)
        st.ids.copy_(torch.randint(0, cfg.vocab, (B,), generator=torch.Generator().manual_seed(4321)).cuda())
        st.set_sampling(temperature=0.7, top_k=50, top_p=0.9, seeds=torch.arange(B), offsets=0)
        st.sample = True  # one stack, two graphs: the step reads the flag while it is captured
        st.graph = None
        g_on, n_on = st.capture(), st.launches_per_step
        st.sample = False
        st.graph = None
        g_off, n_off = st.capture(), st.launches_per_step
        on, off = [], []
        for _ in range(args.rounds):
            on.append(step_ms(st, g_on, ctx, K, W))
            off.append(step_ms(st, g_off, ctx, K, W))
        st.sample = True
        ms_on, ms_off = statistics.median(on), statistics.median(off)
        out["batches"][str(B)] = {"ms_per_step_sampled": round(ms_on, 4), "ms_per_step_greedy": round(ms_off, 4),
                                  "cost_pct": round(100 * (ms_on - ms_off) / ms_off, 2),
                                  "ms_all_sampled": [round(v, 4) for v in on], "ms_all_greedy": [round(v, 4) for v in off],
                                  "launches_per_step": [n_on, n_off]}
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
