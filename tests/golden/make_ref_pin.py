"""Generate tests/golden/ref_pin.npz: what the reference's own GPU code computes on the inputs of tests/test_ref_pin_gpu.py.

Needs a CUDA device and oracle/_ref/libdashinfer_ref.so (python oracle/build_ref.py, from the reference sources):
    python tests/golden/make_ref_pin.py
Stored per case (inputs are regenerated from the tests' seeds):
  append_m{mode}_s{span}_{k,v,q}     sha256 of the K / V span pools and the last Q gather written by DecoderCacheAppendLauncher
  attn_m{mode}_c{case}_{k,v}         sha256 of the pools the same launcher writes for an attention case
  attn_m{mode}_c{case}_out           span::Run's output on those pools, bf16 bits as uint16 [B, nH * 128]
  ctx_m{mode}_s{span}_q{seq}         sha256 of the K pool written by ContextSpanCopyLauncher
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
for p in (ROOT, os.path.join(ROOT, "dash-infer_b200", "python"), os.path.dirname(HERE)):
    sys.path.insert(0, p)

from oracle import kvcache_ref as KV  # noqa: E402
from oracle import ref_lib as RL  # noqa: E402
import test_ref_pin_gpu as T  # noqa: E402

MODES = [KV.QUANT_NONE, KV.QUANT_I8, KV.QUANT_U4]


def main():
    lib = RL.load()
    assert lib is not None, "oracle/_ref/libdashinfer_ref.so is not built"
    out = {}

    def ref_append(cache, qkv, pos):
        nH = cache.cfg.n_heads
        q = torch.empty(qkv.shape[0], nH * 128, dtype=torch.bfloat16, device="cuda")
        RL.cache_append(lib, cache.k_tab, cache.v_tab, q, qkv, pos, nH, cache.cfg.n_groups, cache.cfg.span_len, cache.max_spans,
                        cache.cfg.quant_mode)
        return q

    for mode in MODES:
        for span in (16, 32, 64, 128):
            cache, q, _ = T.append_tokens(ref_append, mode, span, **T.APPEND)
            key = "append_m%d_s%d" % (mode, span)
            out[key + "_k"], out[key + "_v"], out[key + "_q"] = T.digest(cache.k_pool), T.digest(cache.v_pool), T.digest(q)
        for case in range(len(T.CASES)):
            lens, nH, nG, span = T.CASES[case]
            cache, q_last, _ = T.attention_inputs(ref_append, mode, case)
            o = torch.empty_like(q_last)
            RL.span_attn(lib, o, q_last, cache.k_tab, cache.v_tab, lens, nH, nG, span, cache.max_spans, mode, 1.0 / np.sqrt(128))
            torch.cuda.synchronize()
            key = "attn_m%d_c%d" % (mode, case)
            out[key + "_k"], out[key + "_v"] = T.digest(cache.k_pool), T.digest(cache.v_pool)
            out[key + "_out"] = o.view(torch.int16).cpu().numpy().view(np.uint16)
        for span, seq in ((16, 64), (32, 96), (64, 64), (128, 384)):
            cache, src = T.context_copy_inputs(mode, span, seq)
            RL.context_span_copy(lib, cache.k_tab[0], src, cache.cfg.n_groups, span, seq, mode)
            torch.cuda.synchronize()
            out["ctx_m%d_s%d_q%d" % (mode, span, seq)] = T.digest(cache.k_pool)
    dst = os.environ.get("B2_REF_PIN_OUT", os.path.join(HERE, "ref_pin.npz"))
    np.savez_compressed(dst, **{k: np.asarray(v) for k, v in out.items()})
    print("wrote", dst, len(out), "entries")


if __name__ == "__main__":
    main()
