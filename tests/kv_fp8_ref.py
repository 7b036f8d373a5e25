"""CPU restatement of the fp8-e4m3 KV cache (B2_KV_FP8): row quantizer, span layout, a span cache mirror and the decoder
oracle's cache read-back.  Used by tests/test_kv_fp8_oracle.py and tests/test_kv_fp8_gpu.py.

The mode is an extension of the project (span::QuantMode has no fp8 value), so its contract is stated here:
  * span layout = the I8 layout: [n_groups, span_len, 128] e4m3fn codes, then [n_groups, span_len] {f32 zero, f32 scale},
    zero always 0.0;
  * per (token, kv-head) row of 128 values x (the values the FT cache would hold):
        scale = max(max|x|, 1e-12) / 448,  r = 1 / scale   (IEEE fp32)
        code  = e4m3(x * r)                                (fp32 product, round to nearest even, saturating to +-448)
    the same convention as b2_quant_fp8, so the device's bytes are reproduced bit for bit;
  * dequantized value = float(e4m3(code)) * scale.
"""
import numpy as np
import torch

from oracle import kvcache_ref as KV

QUANT_FP8 = 3  # B2_KV_FP8
HEAD = KV.HEAD
E4M3_MAX = np.float32(448.0)


def span_bytes(span_len, n_groups, head=HEAD):
    return span_len * n_groups * head + 2 * span_len * n_groups * 4


def decode(codes):
    """e4m3fn bytes (uint8) -> float32 values."""
    return torch.from_numpy(np.ascontiguousarray(codes, np.uint8)).view(torch.float8_e4m3fn).float().numpy()


def quant_rows(x):
    """x: fp32 [..., HEAD].  Returns (codes uint8 [..., HEAD], zero f32 [...] (all 0), scale f32 [...])."""
    x = np.asarray(x, np.float32)
    amax = np.abs(x).max(axis=-1)
    scale = (np.maximum(amax, np.float32(1e-12)) / E4M3_MAX).astype(np.float32)
    r = (np.float32(1) / scale).astype(np.float32)
    y = (x * r[..., None]).astype(np.float32)
    # satfinite: torch's e4m3fn conversion turns values beyond the format into NaN, the device clamps them to +-448
    y = np.clip(y, -E4M3_MAX, E4M3_MAX)
    codes = torch.from_numpy(np.ascontiguousarray(y)).to(torch.float8_e4m3fn).view(torch.uint8).numpy()
    return codes, np.zeros_like(scale), scale


def dequant_rows(codes, scale):
    return decode(codes) * scale[..., None]


class SpanCacheFp8Ref(KV.SpanCacheRef):
    """KV.SpanCacheRef for B2_KV_FP8 spans (same span list per sequence, same attention_ref)."""

    def __init__(self, span_len, n_groups, head=HEAD):
        self.mode, self.span_len, self.n_groups, self.head, self.ft = QUANT_FP8, span_len, n_groups, head, None
        self.nbytes = span_bytes(span_len, n_groups, head)
        self.spans = []

    def _views(self, buf):
        S, G, H = self.span_len, self.n_groups, self.head
        return buf[: S * G * H].reshape(G, S, H), buf[S * G * H:].view(np.float32).reshape(G, S, 2)

    def append(self, b, pos, rows):
        si, p = pos // self.span_len, pos % self.span_len
        self._ensure(b, si + 1)
        codes, prm = self._views(self.spans[b][si])
        q, z, s = quant_rows(rows)
        codes[:, p, :] = q
        prm[:, p, 0] = z
        prm[:, p, 1] = s

    def dense(self, b, length):
        S, G, H = self.span_len, self.n_groups, self.head
        out = np.zeros((G, length, H), np.float32)
        for si in range((length + S - 1) // S):
            n = min(S, length - si * S)
            codes, prm = self._views(self.spans[b][si])
            out[:, si * S: si * S + n] = dequant_rows(codes[:, :n], prm[:, :n, 1])
        return out


def decoder_ref(stack):
    """oracle.decoder_ref.RefDecoder for a DecodeStack(kv="fp8"): the cache hands back fp8-dequantized K/V rows."""
    from oracle import decoder_ref as DR
    ref = DR.from_stack(stack, KV.QUANT_NONE)

    def store(rows):
        q, _, s = quant_rows(rows.numpy().astype(np.float32))
        return torch.from_numpy(dequant_rows(q, s))

    ref._store = store
    ref.kv_mode = QUANT_FP8
    return ref
