"""Cost of sampling under tensor parallelism on one GPU (b2_sample_shard, graph-replayed), against b2_sample on the whole
row and the greedy vocab-split argmax.

For [B, 152064] bf16 logits, B in {1, 16, 64}, P in {2, 4, 8} even shards, at (t 0.7, k 50, p 0.9) and at t = 1 without
limits, it prints one JSON line per case:
  phase_us      µs of each phase kernel on rank 0's shard (records from a real run of every rank), and the merge
  sum_us        their sum: one rank's kernel time per step, without the exchanges
  sample_us     b2_sample on the whole rows
  argmax_us     b2_argmax_shard + b2_argmax_merge on rank 0's shard (the greedy TP step's kernels)
  allgather_us  b2_allgather of each phase's records between P loopback communicators on this one GPU (every rank on
                its own stream): a loopback figure, not an NVLink one
The step cost under real tensor parallelism needs >= 2 GPUs and is not measured here.

Usage: python tools/sample_tp_bench.py [--reps 200]"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "dash-infer_b200", "python"))
from b200spark import ops  # noqa: E402

N = 152064
PHASES = 6


def _time(fn, reps):
    """µs per call of fn, replayed from a CUDA graph of `reps` calls"""
    fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(reps):
            fn()
    g.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    best = float("inf")
    for _ in range(5):
        e0.record()
        g.replay()
        e1.record()
        torch.cuda.synchronize()
        best = min(best, e0.elapsed_time(e1) * 1e3 / reps)
    return best


def _params(B, t, k, p):
    return (torch.full((B,), t, device="cuda"), torch.full((B,), k, dtype=torch.int32, device="cuda"),
            torch.full((B,), p, device="cuda"), torch.arange(B, dtype=torch.int64, device="cuda") + 7,
            torch.zeros(B, dtype=torch.int64, device="cuda"))


def _loopback_allgather_us(P, nbytes, reps):
    comms = ops.Comm.connect_local([ops.Comm(q, P, nbytes) for q in range(P)])
    streams = [torch.cuda.Stream() for _ in range(P)]
    src = [torch.zeros(nbytes, dtype=torch.uint8, device="cuda") for _ in range(P)]
    dst = [torch.empty(P, nbytes, dtype=torch.uint8, device="cuda") for _ in range(P)]
    for q in range(P):
        with torch.cuda.stream(streams[q]):
            comms[q].allgather(src[q], dst[q])
    torch.cuda.synchronize()
    graphs = [torch.cuda.CUDAGraph() for _ in range(P)]
    for q in range(P):
        with torch.cuda.graph(graphs[q], stream=streams[q]):
            for _ in range(reps):
                comms[q].allgather(src[q], dst[q])
    cur = torch.cuda.current_stream()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    best = float("inf")
    for _ in range(3):
        e0.record(cur)
        for q in range(P):
            streams[q].wait_event(e0)
            with torch.cuda.stream(streams[q]):
                graphs[q].replay()
        for q in range(P):
            cur.wait_stream(streams[q])
        e1.record(cur)
        torch.cuda.synchronize()
        best = min(best, e0.elapsed_time(e1) * 1e3 / reps)
    for c in comms:
        c.check_error()
    return best


def bench(B, P, t, k, p, reps):
    gen = torch.Generator(device="cuda").manual_seed(B + P)
    logits = (torch.randn(B, N, generator=gen, device="cuda") * 2).to(torch.bfloat16)
    prm = _params(B, t, k, p)
    s = N // P
    bounds = [q * s for q in range(P)] + [N]
    bufs = [ops.sample_tp_buffers(B, P) for _ in range(P)]
    prms = [[x.clone() for x in prm] for _ in range(P)]
    for ph in range(PHASES):  # one real run of every rank: rank 0's all-gathered records of every phase
        for q in range(P):
            ops.sample_shard(ph, logits[:, bounds[q]:bounds[q + 1]], bounds[q], N, *prms[q], bufs[q]["state"],
                             bufs[q]["all"][ph - 1] if ph else None, out=bufs[q]["rec"][ph], nranks=P)
        for q in range(P):
            for r in range(P):
                bufs[q]["all"][ph][r].copy_(bufs[r]["rec"][ph].view(-1))
    b0, shard = bufs[0], logits[:, :bounds[1]]

    def prefix(m):  # rank 0's phases 0 .. m - 1 (m = PHASES + 1: and the merge), on the gathered records of the real run
        def fn():
            for ph in range(min(m, PHASES)):
                ops.sample_shard(ph, shard, 0, N, *prms[0], b0["state"], b0["all"][ph - 1] if ph else None,
                                 out=b0["rec"][ph], nranks=P)
            if m > PHASES:
                ops.sample_shard_merge(b0["all"][PHASES - 1], b0["state"], prms[0][4], out=ids)
        return fn

    ids = torch.empty(B, dtype=torch.int64, device="cuda")
    cum = [0.0] + [_time(prefix(m), reps) for m in range(1, PHASES + 2)]
    phase_us = [round(max(cum[m + 1] - cum[m], 0.0), 2) for m in range(PHASES + 1)]
    offs = prm[4].clone()
    sample_us = _time(lambda: ops.sample(logits, *prm[:4], offs, out=ids), reps)
    li, lv = torch.empty(B, dtype=torch.int64, device="cuda"), torch.empty(B, dtype=torch.float32, device="cuda")
    ai, av = torch.zeros(P, B, dtype=torch.int64, device="cuda"), torch.zeros(P, B, dtype=torch.float32, device="cuda")

    def argmax_fn():
        ops.argmax_shard(shard, 0, li, lv)
        ops.argmax_merge(av, ai, out=ids)
    argmax_us = _time(argmax_fn, reps)
    gather = {ph: round(_loopback_allgather_us(P, B * ops.sample_shard_record_bytes(ph), 50), 2) for ph in range(PHASES)}
    return {"B": B, "P": P, "params": {"t": t, "k": k, "p": p},
            "phase_us": dict(zip([f"phase{ph}" for ph in range(PHASES)] + ["merge"], phase_us)),
            "sum_us": round(cum[-1], 2), "sample_us": round(sample_us, 2), "argmax_us": round(argmax_us, 2),
            "allgather_us": {f"phase{ph} ({B * ops.sample_shard_record_bytes(ph)} B per rank, loopback)": v
                             for ph, v in gather.items()}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--out", default=None, help="also write the JSON lines to this file")
    a = ap.parse_args()
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i",
                                str(torch.cuda.current_device())], capture_output=True, text=True).stdout.strip()
    except OSError:
        power = "unknown"
    lines = [json.dumps({"device": torch.cuda.get_device_name(), "power_limit": power, "n": N, "dtype": "bf16",
                         "step_cost_under_real_tp": "not measured (needs >= 2 GPUs)"})]
    print(lines[-1], flush=True)
    for B in (1, 16, 64):
        for P in (2, 4, 8):
            for t, k, p in ((0.7, 50, 0.9), (1.0, 0, 1.0)):
                lines.append(json.dumps(bench(B, P, t, k, p, a.reps)))
                print(lines[-1], flush=True)
    if a.out:
        with open(a.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
