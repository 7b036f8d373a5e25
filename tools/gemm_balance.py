"""Time the batch 17-64 wgmma GEMMs of one Qwen2-7B int4 layer against their work schedule (run on the GPU box).

  python tools/gemm_balance.py [--m 17,32,64] [--shapes gateup,down,qkv,o] [--env B2_GEMM_TC_MAX_SPLIT=4 ...]

For every shape and batch it replays, from a CUDA graph, one launch per layer over enough layers' weights to overflow L2,
times the replays with CUDA events and prints us per launch, GB/s of the bytes the GEMM must move, the grid and the largest
number of 64-k tiles one CTA streams (tests/tc_schedule.py; cluster = CTAs per thread-block cluster as the handle planned
it, 1 for the workspace split-K or no split).  Then it fits time = fixed + rate * tiles over the shapes of each
batch: the per-launch fixed cost and the per-tile cost of the main loop.  A shape is NAME or NAME=KxN (p: gate/up pair),
e.g. gate264=3584x16896p.  Writes nothing."""
import argparse
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "dash-infer_b200", "python"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

SHAPES = {"gateup": (3584, 18944, True), "down": (18944, 3584, False), "qkv": (3584, 4608, False), "o": (3584, 3584, False)}


def parse_shape(s):
    if "=" not in s:
        return s, SHAPES[s]
    name, dims = s.split("=")
    pair = dims.endswith("p")
    K, N = dims.rstrip("p").split("x")
    return name, (int(K), int(N), pair)


def handles(K, N, pair, M, min_bytes, torch, ops):
    g = torch.Generator(device="cuda").manual_seed(0)

    def wset():
        q = torch.randint(0, 256, (K, (N + 1) // 2), dtype=torch.uint8, device="cuda", generator=g)
        s = (torch.rand(1, N, device="cuda", generator=g) * 1e-3 + 1e-3).to(torch.bfloat16)
        z = torch.full((1, N), 8.0, device="cuda").to(torch.bfloat16)
        return q, s, z
    per = K * N // 2 * (2 if pair else 1)
    nw = max(4, min(28, -(-min_bytes // per)))
    hs = []
    for _ in range(nw):
        h = ops.GemmWQ(K, N, 4, -1, max_m=M, pair=pair)
        hs.append(h.prepare_swiglu(*wset(), *wset()) if pair else h.prepare(*wset()))
    return hs


def time_launch(hs, M, K, N, torch, ops, reps):
    a = (torch.randn(M, K, device="cuda") * 0.1).to(torch.bfloat16)
    out = torch.empty(M, N, dtype=torch.bfloat16, device="cuda")
    ws = ops.Workspace()
    for h in hs:
        h(a, ws, out=out)
    torch.cuda.synchronize()
    loops = max(1, 64 // len(hs))
    graph, s = torch.cuda.CUDAGraph(), torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s), torch.cuda.graph(graph, stream=s):
        for _ in range(loops):
            for h in hs:
                h(a, ws, out=out)
    torch.cuda.current_stream().wait_stream(s)
    graph.replay()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        graph.replay()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1) * 1e3 / (loops * len(hs)))
    return float(np.median(ts)), float(np.min(ts)), float(np.max(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--m", default="17,32,64")
    ap.add_argument("--shapes", default="gateup,down,qkv,o")
    ap.add_argument("--env", action="append", default=[], help="KEY=VALUE set before the handles are made")
    ap.add_argument("--min-mb", type=int, default=256, help="weights cycled per shape (L2 is 50 MB)")
    ap.add_argument("--reps", type=int, default=9)
    args = ap.parse_args()
    for kv in args.env:
        k, v = kv.split("=", 1)
        os.environ[k] = v
    import torch
    from b200spark import ops
    import tc_schedule
    if not torch.cuda.is_available():
        sys.exit("gemm_balance.py times the GPU kernels: no CUDA device")
    prop = torch.cuda.get_device_properties(0)
    sms = prop.multi_processor_count
    max_split = int(os.environ.get("B2_GEMM_TC_MAX_SPLIT", tc_schedule.MAX_SPLIT))
    persist = os.environ.get("B2_GEMM_TC_PERSIST", "1") != "0"
    print(f"# {prop.name}, {sms} SMs, env {args.env or 'default'}")
    shapes = [parse_shape(s) for s in args.shapes.split(",")]
    for M in [int(m) for m in args.m.split(",")]:
        pts = []
        for name, (K, N, pair) in shapes:
            hs = handles(K, N, pair, M, args.min_mb << 20, torch, ops)
            med, lo, hi = time_launch(hs, M, K, N, torch, ops, args.reps)
            NG = (N + 63) // 64 if pair else (N + 127) // 128
            pl = tc_schedule.plan(NG, (K + 63) // 64, sms, max_split, persist)
            tiles = pl.max_tiles()
            gbs = hs[0].algo_bytes(M) / (med * 1e-6) / 1e9
            print(f"{name:8s} M={M:3d} K={K:5d} N={N:5d}{'x2' if pair else '  '} layers={len(hs):2d}  {med:7.2f} us "
                  f"[{lo:.2f}, {hi:.2f}]  {gbs:7.1f} GB/s  grid={pl.grid:3d} rounds={pl.rounds} slices={pl.S} cluster={hs[0].tc_cluster()} head={pl.h:2d} "
                  f"max_tiles/CTA={tiles:4d}", flush=True)
            pts.append((tiles, med))
            del hs
            torch.cuda.empty_cache()
        if len({t for t, _ in pts}) > 1:
            x, y = np.array(pts, dtype=np.float64).T
            rate, fixed = np.polyfit(x, y, 1)
            print(f"fit M={M}: time = {fixed:.2f} us fixed + {rate:.4f} us per tile per CTA")


if __name__ == "__main__":
    main()
