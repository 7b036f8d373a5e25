"""GPU: b2_penalize against the reference's own logits processor (LogitsProcessor, beam_search.cu, compiled with its
fast-math flags), pinned in tests/golden/penalty_pin.npz by tests/golden/make_penalty_pin.py on the inputs of
test_penalty_gpu.py::test_matches_restatement.

Bit for bit, except the two differences include/b200spark.h documents:
- -0 becomes +0 in the reference in every column outside the history when FT(0 * frequency) is -0; this test
  predicts that set from the inputs, and the differing columns must be exactly those;
- where both results are NaN, their bits may differ (the reference writes canonical NaNs).
Nothing else may differ: not the repetition quotient (the reference runs the same __hdiv), not the fp32 penalty sum."""
import os
import zlib

import numpy as np
import pytest
import torch

import penalty_ref as P

pytestmark = pytest.mark.gpu

PIN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "penalty_pin.npz")


@pytest.fixture(scope="module")
def pin():
    return np.load(PIN)


def reference_bits(pin, key, x_bits):
    out = x_bits.reshape(-1).copy()
    pos = np.cumsum(pin[key + "_idx"].astype(np.int64))
    out[pos] = pin[key + "_bits"]
    return out.reshape(x_bits.shape)


@pytest.mark.parametrize("ft,n,rows", P.CASES)
def test_matches_the_reference_processor(pin, ft, n, rows):
    from b200spark import ops
    hists, prompts, prm, x = P.case(ft, n, rows)
    xb = P.bits(x, ft)
    key = "%s_%d_%d" % (ft, n, rows)
    assert zlib.crc32(xb.tobytes()) == int(pin[key + "_crc"]), "the inputs are not the ones the pin was made from"
    ref = reference_bits(pin, key, xb)
    hist = ops.TokenHistory(rows, 256, n)
    for r, (h, p) in enumerate(zip(hists, prompts)):
        hist.load(r, h, p)
    pen = ops.Penalties(rows)
    for k in P.neutral(0):
        getattr(pen, k).copy_(torch.tensor(prm[k]))
    y = torch.from_numpy(xb.view(np.int16).copy()).cuda().view(P.FTS[ft])
    ops.penalize(y, hist, pen)
    got = y.view(torch.int16).cpu().numpy().view(np.uint16)

    nan_got, nan_ref = np.isnan(P.values(got, ft)), np.isnan(P.values(ref, ft))
    differ = (got != ref) & ~(nan_got & nan_ref)
    # the documented -0 -> +0 columns: input -0, not in the row's history nor banned, and a -0 penalty for a count of 0
    neg_zero = np.zeros_like(differ)
    for r in range(rows):
        pen0 = P.rn(P.penalty_sum(0, prm["frequency"][r], prm["presence"][r]), ft)[()]
        if pen0 == 0 and np.signbit(pen0):
            cols = (xb[r] == 0x8000)
            cols[[t for t in set(int(t) for t in hists[r]) if 0 <= t < n]] = False
            eos = int(prm["eos_id"][r])
            if len(hists[r]) < prm["min_length"][r] and 0 <= eos < n:
                cols[eos] = False  # banned, in both
            neg_zero[r] = cols
    assert np.array_equal(differ, neg_zero), [(int(r), int(c), hex(got[r, c]), hex(ref[r, c]), hex(xb[r, c]))
                                              for r, c in np.argwhere(differ != neg_zero)[:8]]
    assert np.all(ref[neg_zero] == 0x0000) and np.all(got[neg_zero] == 0x8000)

