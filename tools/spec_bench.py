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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--ctx", type=int, default=2048)
    args = ap.parse_args()
    name, power = gpu_info()
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
