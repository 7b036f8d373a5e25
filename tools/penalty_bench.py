"""Cost of the logits processor (b2_penalize) on one GPU.

  * b2_penalize on [B, 152064] bf16 logits at B = 1, 8, 64, over history lengths 1, 2K, 32K and 128K, each with all ids
    distinct and with 64 distinct ids (heavy repeats), at repetition 1.1, presence 0.5, frequency 0.5 and a no-repeat
    3-gram: µs per launch, CUDA events over launches replayed from a CUDA graph (bench.time_kernel_loop), next to b2_argmax
    on the same row;
  * the Qwen2-7B step (bench.py's workload: int4 per-channel, bf16 KV, ctx 2048) with penalties on (a 2048-token history
    per sequence, the parameters above) against the same step without, at B = 64, 8, 1: one set of weights and caches, a
    graph of each, alternated in `--rounds` rounds, the history restored before every run; medians reported;
  * the card's name and power limit, read in the same run.
Prints one JSON line.  Usage (the DESIGN.md §3.9 tables): python tools/penalty_bench.py --steps 20 --warmup 5 --rounds 5

--tokens: the verify-step form (b2_penalize_tokens):
  * µs per launch on [B*T, 152064] bf16 rows, graph-replayed as above, at B = 1, 8, 64, T = 4, 8, 16, chains and width-4
    trees (node t's parent: (t - 1) // 4), over histories of 2K and 32K tokens, all distinct and 64 distinct, at the
    parameters above; next to b2_penalize on B rows and on B*T rows of the same histories;
  * the cost in a Qwen2-7B int4 verify step (ctx 2048, chain, T = 4 / 8 / 16, B = 1 and 8): the captured step with one
    b2_penalize_tokens launch over a 2K-token history appended at its end, against the plain step, alternated in
    `--rounds` rounds; medians and the spread.  The appended launch runs on logits the step has already consumed, so it
    measures cost only, not a functional penalised step.
Usage (the DESIGN.md §5 table): python tools/penalty_bench.py --tokens --steps 30 --warmup 5 --rounds 5
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

HISTORY = [1, 2048, 32768, 131072]
PARAMS = dict(repetition=1.1, presence=0.5, frequency=0.5, no_repeat_ngram=3)


def kernels_us(B, rounds):
    g = torch.Generator(device="cuda").manual_seed(B)
    bufs = [(torch.randn(B, VOCAB, generator=g, device="cuda") * 3).to(torch.bfloat16) for _ in range(4)]
    ids = torch.empty(B, dtype=torch.int64, device="cuda")
    pen = ops.Penalties(B).set(**PARAMS)
    fns = {"argmax": [lambda x=x: ops.argmax(x, out=ids) for x in bufs]}
    hists = {}
    for L in HISTORY:
        for distinct in (L, min(L, 64)):
            h = ops.TokenHistory(B, L, VOCAB)
            for b in range(B):
                toks = torch.randint(0, VOCAB, (distinct,), generator=torch.Generator().manual_seed(b))
                h.load(b, toks.repeat((L + distinct - 1) // distinct)[:L], L // 2)
            hists[(L, distinct)] = h
            fns["penalize[L=%d,distinct=%d]" % (L, distinct)] = [lambda x=x, h=h: ops.penalize(x, h, pen) for x in bufs]
    res = {name: [] for name in fns}
    for _ in range(rounds):  # alternated
        for name, f in fns.items():
            res[name].append(bench.time_kernel_loop(f, 25, torch) * 1e6)
    del hists
    return {name: round(statistics.median(v), 2) for name, v in res.items()}


def step_ms(st, graph, ctx, K, W, snap):
    st.graph = graph
    bench.rewind(st, ctx)
    if snap is not None:
        st.history.restore(snap)
    ms, _ = bench.timed_steps(st, K, W, torch, None, 1)
    return ms / K


def tree_parents(B, T):
    return torch.tensor([[0] + [(t - 1) // 4 for t in range(1, T)]] * B, dtype=torch.int32, device="cuda")


def tokens_kernels_us(B, rounds):
    g = torch.Generator(device="cuda").manual_seed(B)
    pen = ops.Penalties(B).set(**PARAMS)
    pen_bt = ops.Penalties(B * 16).set(**PARAMS)
    res = {}
    for L in (2048, 32768):
        for distinct in (L, 64):
            h = ops.TokenHistory(B, L + 16, VOCAB)
            hbt = ops.TokenHistory(B * 16, L + 16, VOCAB)
            for b in range(B):
                toks = torch.randint(0, VOCAB, (distinct,), generator=torch.Generator().manual_seed(b))
                toks = toks.repeat((L + distinct - 1) // distinct)[:L]
                h.load(b, toks, L // 2)
                for t in range(16):
                    hbt.load(b * 16 + t, toks, L // 2)
            key = "L=%d,distinct=%d" % (L, distinct)
            fns = {}
            bufs = [(torch.randn(B * 16, VOCAB, generator=g, device="cuda") * 3).to(torch.bfloat16) for _ in range(2)]
            fns["penalize[B]"] = [lambda x=x: ops.penalize(x[:B], h, pen) for x in bufs]
            for T in (4, 8, 16):
                tk = torch.randint(0, VOCAB, (B, T), generator=g, device="cuda")
                par = tree_parents(B, T)
                fns["penalize[B*T],T=%d" % T] = [lambda x=x, T=T: ops.penalize(x[:B * T], hbt, pen_bt) for x in bufs]
                fns["tokens_chain,T=%d" % T] = [lambda x=x, T=T, tk=tk: ops.penalize_tokens(x[:B * T], h, pen, tk) for x in bufs]
                fns["tokens_tree,T=%d" % T] = [lambda x=x, T=T, tk=tk, par=par: ops.penalize_tokens(x[:B * T], h, pen, tk, par)
                                               for x in bufs]
            times = {name: [] for name in fns}
            for _ in range(rounds):  # alternated
                for name, f in fns.items():
                    times[name].append(bench.time_kernel_loop(f, 25, torch) * 1e6)
            res[key] = {name: round(statistics.median(v), 2) for name, v in times.items()}
            del h, hbt, bufs
            torch.cuda.empty_cache()
    return res


def tokens_step(args, out):
    cfg = model.QWEN2_7B
    K, W = args.steps, max(args.warmup, 3)
    gen = torch.Generator(device="cuda").manual_seed(9)
    hist = ops.TokenHistory(8, 2048 + 32, cfg.vocab)
    for b in range(8):
        hist.load(b, torch.randint(0, cfg.vocab, (2048,), generator=torch.Generator().manual_seed(b)), 1024)
    pen = ops.Penalties(8).set(**PARAMS)
    out["step"] = []
    for T in (4, 8, 16):
        st = model.DecodeStack(cfg, 8, args.ctx + 64, wbits=4, group=-1, kv="none", span=128, q_len=T, layers=args.layers)
        st.set_context(args.ctx)
        plain = st._step_ops
        for B in (8, 1):
            st.set_batch(B)
            h, p = hist.view(B), pen.view(B)
            st.tokens.copy_(torch.randint(0, cfg.vocab, st.tokens.shape, generator=gen, device="cuda"))
            lo, ln, tk = st.lens_old.clone(), st.lens_new.clone(), st.tokens.clone()
            st._step_ops = plain
            g_off = st.capture()
            st._step_ops = lambda: (plain(), ops.penalize_tokens(st.logits, h, p, st.tokens))[0]
            g_on = st.capture()

            def ms(g):
                def step():
                    g.replay()
                    st.lens_old.copy_(lo); st.lens_new.copy_(ln); st.tokens.copy_(tk)
                for _ in range(W):
                    step()
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(K):
                    step()
                e1.record()
                torch.cuda.synchronize()
                return e0.elapsed_time(e1) / K

            on, off = [], []
            for _ in range(args.rounds):
                on.append(ms(g_on))
                off.append(ms(g_off))
            m_on, m_off = statistics.median(on), statistics.median(off)
            out["step"].append({"q_len": T, "batch": B, "ms_plain": round(m_off, 4), "ms_with_penalize_tokens": round(m_on, 4),
                                "cost_pct": round(100 * (m_on - m_off) / m_off, 2),
                                "ms_all_plain": [round(v, 4) for v in off], "ms_all_with": [round(v, 4) for v in on]})
            print(json.dumps(out["step"][-1]), file=sys.stderr, flush=True)
        st._step_ops = plain
        del st
        torch.cuda.empty_cache()


def tokens_main(args):
    name, power = gpu_info()
    out = {"gpu": name, "power_limit": power, "params": PARAMS, "rounds": args.rounds, "kernels_us": {},
           "model": model.QWEN2_7B.name, "ctx": args.ctx, "steps": args.steps}
    for B in (1, 8, 64):
        out["kernels_us"][str(B)] = tokens_kernels_us(B, args.rounds)
        print(json.dumps({str(B): out["kernels_us"][str(B)]}), file=sys.stderr, flush=True)
    tokens_step(args, out)
    print(json.dumps(out), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--ctx", type=int, default=2048)
    ap.add_argument("--batches", default="64,8,1")
    ap.add_argument("--rounds", type=int, default=5, help="alternations of the measurements with and without penalties")
    ap.add_argument("--layers", type=int, default=None, help="debug: fewer layers (not a Qwen2-7B number)")
    ap.add_argument("--tokens", action="store_true", help="b2_penalize_tokens: kernel times and the cost in a verify step")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "penalty_bench measures on the GPU; there is no CPU fallback"
    if args.tokens:
        return tokens_main(args)
    name, power = gpu_info()
    batches = [int(b) for b in args.batches.split(",")]
    K, W, ctx = args.steps, max(args.warmup, 3), args.ctx
    out = {"gpu": name, "power_limit": power, "kernels_us": {}, "model": model.QWEN2_7B.name, "ctx": ctx, "steps": K,
           "rounds": args.rounds, "params": PARAMS, "batches": {}}
    for B in (1, 8, 64):
        out["kernels_us"][str(B)] = kernels_us(B, args.rounds)
    cfg = model.QWEN2_7B
    st = model.DecodeStack(cfg, max(batches), ctx + W + K + 16, wbits=4, group=-1, kv="none", span=128, layers=args.layers,
                           penalties=True)
    st.set_context(ctx)
    for b in range(max(batches)):
        toks = torch.randint(0, cfg.vocab, (ctx,), generator=torch.Generator().manual_seed(b))
        st.set_history(b, toks, ctx // 2)
    for B in batches:
        st.set_batch(B)
        st.ids.copy_(torch.randint(0, cfg.vocab, (B,), generator=torch.Generator().manual_seed(4321)).cuda())
        st.set_penalties(**PARAMS)
        snap = st.history.snapshot()
        st.pen = True  # one stack, two graphs: the step reads the flag while it is captured
        st.graph = None
        g_on, n_on = st.capture(), st.launches_per_step
        st.pen = False
        st.graph = None
        g_off, n_off = st.capture(), st.launches_per_step
        st.pen = True
        on, off = [], []
        for _ in range(args.rounds):
            on.append(step_ms(st, g_on, ctx, K, W, snap))
            off.append(step_ms(st, g_off, ctx, K, W, None))
        st.history.restore(snap)
        ms_on, ms_off = statistics.median(on), statistics.median(off)
        out["batches"][str(B)] = {"ms_per_step_penalized": round(ms_on, 4), "ms_per_step_plain": round(ms_off, 4),
                                  "cost_pct": round(100 * (ms_on - ms_off) / ms_off, 2),
                                  "ms_all_penalized": [round(v, 4) for v in on], "ms_all_plain": [round(v, 4) for v in off],
                                  "launches_per_step": [n_on, n_off]}
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
