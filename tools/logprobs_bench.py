"""Cost of the decode step's log-probabilities on one GPU.

  * b2_logprobs with n_top 0 / 1 / 10 against b2_argmax on [B, 152064] bf16 logits at B = 1, 8, 64: µs per launch, CUDA events
    over launches replayed from a CUDA graph (bench.time_kernel_loop), cycling through 4 logits buffers.  At B = 1 and 8 the
    four buffers (1.2 / 9.7 MB) stay in the 50 MB L2, as the logits of a decode step do right after lm_head wrote them; at
    B = 64 (78 MB) they come mostly from HBM;
  * the Qwen2-7B step (bench.py's workload: int4 per-channel, bf16 KV, ctx 2048) with logprobs=0 and logprobs=10 at B = 64, 8,
    1: one stack, weights and caches, a graph of each, alternated in `--rounds` rounds; medians reported;
  * the card's name and power limit, read in the same run.
Prints one JSON line.  Usage (the DESIGN.md §3.7 table): python tools/logprobs_bench.py --steps 30 --warmup 5
"""
import argparse
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

VOCAB = 152064


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=20).stdout.strip()
        name, power = [x.strip() for x in r.split(",")]
        return name, power
    except Exception:
        return torch.cuda.get_device_name(0), None


def kernels_us(B, rounds):
    g = torch.Generator(device="cuda").manual_seed(B)
    bufs = [(torch.randn(B, VOCAB, generator=g, device="cuda") * 3).to(torch.bfloat16) for _ in range(4)]
    ids = torch.empty(B, dtype=torch.int64, device="cuda")
    outs = {k: ops._lp_outputs(B, k, "cuda", None) for k in (0, 1, 10)}
    fns = {"argmax": [lambda x=x: ops.argmax(x, out=ids) for x in bufs]}
    for k in (0, 1, 10):
        fns["logprobs[n_top=%d]" % k] = [lambda x=x, k=k: ops.logprobs(x, k, out=outs[k]) for x in bufs]
    res = {name: [] for name in fns}
    for _ in range(rounds):  # alternated
        for name, f in fns.items():
            res[name].append(bench.time_kernel_loop(f, 25, torch) * 1e6)
    return {name: round(statistics.median(v), 2) for name, v in res.items()}


def capture(st, n):
    st.logprobs = n
    st.graph = None
    st.capture()
    return st.graph, st.launches_per_step


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
    ap.add_argument("--rounds", type=int, default=5, help="alternations of the with / without-logprobs measurements")
    ap.add_argument("--layers", type=int, default=None, help="debug: fewer layers (not a Qwen2-7B number)")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "logprobs_bench measures on the GPU; there is no CPU fallback"
    name, power = gpu_info()
    batches = [int(b) for b in args.batches.split(",")]
    K, W, ctx = args.steps, max(args.warmup, 3), args.ctx
    out = {"gpu": name, "power_limit": power, "kernels_us": {}, "model": model.QWEN2_7B.name, "ctx": ctx, "steps": K,
           "rounds": args.rounds, "batches": {}}
    for B in (1, 8, 64):
        out["kernels_us"][str(B)] = kernels_us(B, args.rounds)
    cfg = model.QWEN2_7B
    st = model.DecodeStack(cfg, max(batches), ctx + W + K + 16, wbits=4, group=-1, kv="none", span=128, layers=args.layers,
                           logprobs=10)
    st.set_context(ctx)
    for B in batches:
        st.set_batch(B)
        st.ids.copy_(torch.randint(0, cfg.vocab, (B,), generator=torch.Generator().manual_seed(4321)).cuda())
        g_on, n_on = capture(st, 10)
        g_off, n_off = capture(st, 0)
        on, off = [], []
        for _ in range(args.rounds):
            on.append(step_ms(st, g_on, ctx, K, W))
            off.append(step_ms(st, g_off, ctx, K, W))
        ms_on, ms_off = statistics.median(on), statistics.median(off)
        out["batches"][str(B)] = {"ms_per_step_logprobs10": round(ms_on, 4), "ms_per_step_logprobs0": round(ms_off, 4),
                                  "cost_pct": round(100 * (ms_on - ms_off) / ms_off, 2),
                                  "ms_all_logprobs10": [round(v, 4) for v in on], "ms_all_logprobs0": [round(v, 4) for v in off],
                                  "launches_per_step": [n_on, n_off]}
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
