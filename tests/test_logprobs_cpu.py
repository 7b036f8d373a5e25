"""CPU: the log-probability kernels' definitions, bound and argument checks (tests/logprobs_ref.py), without a GPU.

The restated kernel (fp32 arithmetic in the kernel's order) lies within the bound of fp64 log_softmax on every row kind, and
two wrong kernels (logprobs rounded to bf16 as the reference returns them; per-thread sums in bf16) do not; shard records
merged across a vocab split give the whole row's ids and stay within the merge bound; non-finite rows follow torch exactly;
bad arguments return B2_ERR_PARAM before any launch; the kernels keep their per-thread top-10 in registers."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

import glue_ref as G
import logprobs_ref as P

B2_ERR_PARAM = 3


def _rows(n, dt, seed):
    """every ARGMAX_KINDS row and the three logprob kinds, [rows, n] fp32 exact in dt"""
    rng = np.random.default_rng(seed)
    rows = [G.ft_values(G.argmax_row(k, n, rng), dt) for k in G.ARGMAX_KINDS]
    rows += [P.lp_row(k, n, dt, rng) for k in P.LP_KINDS]
    return np.stack(rows)


def _check_restated(x, n, n_top, shards=None, tok_ids=None):
    ids, tlp, tids, tlps = P.restated(x, n, n_top, tok_ids, shards)
    exact, bound = P.lp_bound(x, n, shards)
    want_ids = P.top_order(x, n, max(n_top, 1))
    assert np.array_equal(ids, want_ids[:, 0])
    assert np.array_equal(tids, want_ids[:, :n_top])
    worst = P.lp_ratio(tlps, P.gather(exact, tids), P.gather(bound, tids)) if n_top else 0.0
    tok = want_ids[:, 0] if tok_ids is None else np.asarray(tok_ids)
    ok = (tok >= 0) & (tok < n)
    tok_exact = np.where(ok, P.gather(exact, np.where(ok, tok, 0)[:, None])[:, 0], np.nan)
    tok_bound = np.where(ok, P.gather(bound, np.where(ok, tok, 0)[:, None])[:, 0], 0.0)
    worst = max(worst, P.lp_ratio(tlp, tok_exact, tok_bound))
    return worst


@pytest.mark.parametrize("n", [1, 31, 1025, 151936])
@pytest.mark.parametrize("dt", ["bf16", "fp16"])
def test_bound_holds_on_the_restatement(n, dt):
    """whole rows: the restated kernel's top ids are the argmax order and its logprobs lie within the bound"""
    ft = G.FTS[dt]
    x = _rows(n, ft, seed=n)
    for n_top in P.N_TOPS:
        assert _check_restated(x, n, n_top) <= 1.0, n_top
    tok = np.random.default_rng(1).integers(-3, n + 3, x.shape[0])
    assert _check_restated(x, n, 10, tok_ids=tok) <= 1.0


def test_bound_rejects_wrong_kernels():
    """bf16 logprobs (the reference's FT rounding) and bf16 per-thread sums miss the bound by far"""
    rng = np.random.default_rng(5)
    n = 151936
    x = np.stack([G.ft_values(rng.standard_normal(n) * 3, torch.bfloat16) for _ in range(3)])
    exact, bound = P.lp_bound(x, n)
    for variant in ("ft_lp", "sum_bf16"):
        _, _, tids, tlps = P.restated(x, n, 10, variant=variant)
        ratio = P.lp_ratio(tlps, P.gather(exact, tids), P.gather(bound, tids))
        assert ratio > 4.0, (variant, ratio)


@pytest.mark.parametrize("tp", [2, 4, 8])
def test_merge_of_shard_records(tp):
    """shard records merged = the whole row: ids identical, logprobs within the merge bound, for winners and ties on
    shard edges, NaN in two shards, all -inf; one shard + the merge is the whole-row restatement exactly"""
    n = 4099
    rng = np.random.default_rng(tp)
    x = np.stack([G.tp_row(k, n, tp, rng) for k in G.TP_KINDS] + [P.lp_row(k, n, torch.bfloat16, rng) for k in P.LP_KINDS])
    shards = G.shard_bounds(n, tp)
    tok = rng.integers(0, n, x.shape[0])
    for n_top in (1, 10):
        assert _check_restated(x, n, n_top, shards=shards, tok_ids=tok) <= 1.0
        whole = P.restated(x, n, n_top, tok)
        split = P.restated(x, n, n_top, tok, shards)
        assert np.array_equal(whole[0], split[0]) and np.array_equal(whole[2], split[2])
        one = P.restated(x, n, n_top, tok, [(0, n)])
        for a, b in zip(whole, one):
            assert np.array_equal(a, b, equal_nan=a.dtype.kind == "f")


def test_nonfinite_rows_follow_torch():
    """NaN anywhere, a +inf, all -inf: every logprob NaN; -inf entries beside a finite maximum: -inf; ids in argmax order"""
    inf, nan = np.inf, np.nan
    x = np.array([[1.0, nan, 2.0, 3.0, 0.5], [1.0, inf, 2.0, -inf, 0.0], [-inf] * 5, [1.0, -inf, 2.0, 3.0, -inf],
                  [inf, inf, 0.0, nan, 1.0]], np.float32)
    want = torch.log_softmax(torch.from_numpy(x).double(), -1).float().numpy()
    _, _, tids, tlps = P.restated(x, 5, 5)
    assert np.array_equal(tids, P.top_order(x, 5, 5))
    exact, bound = P.lp_bound(x, 5)
    assert np.array_equal(np.isnan(tlps), np.isnan(P.gather(want, tids)))
    assert P.lp_ratio(tlps, P.gather(exact, tids), P.gather(bound, tids)) <= 1.0
    assert np.isnan(want[:3]).all() and np.isnan(want[4]).all() and np.isinf(want[3, [1, 4]]).all()


def test_argument_checks_without_gpu():
    """every rejected call returns B2_ERR_PARAM before a launch (the addresses are never dereferenced)"""
    from b200spark import _lib
    lib, bf = _lib.lib, _lib.DT_BF16
    A = 1 << 20
    assert lib.b2_logprobs_partial_bytes(0) == lib.b2_logprobs_partial_bytes(1) == 16 + 8
    assert lib.b2_logprobs_partial_bytes(10) == 16 + 80
    assert lib.b2_logprobs_partial_bytes(11) == 0 and lib.b2_logprobs_partial_bytes(-1) == 0
    bad = [
        (A, A, A, A, None, A, 1, 100, 100, 11, bf),       # n_top > 10
        (A, A, None, None, None, A, 1, 100, 100, -1, bf),  # n_top < 0
        (A, A, None, None, None, A, 1, 0, 100, 0, bf),     # n < 1
        (A, A, None, None, None, A, 1, 100, 99, 0, bf),    # ld < n
        (A, A, None, A, None, A, 1, 100, 100, 5, bf),      # top_ids NULL with n_top > 0
        (A, A, A, None, None, A, 1, 100, 100, 5, bf),      # top_lp NULL with n_top > 0
        (A, A, A, A, None, A, 1, 100, 100, 0, bf),         # top outputs with n_top == 0
        (None, None, None, None, None, A, 1, 100, 100, 0, bf),  # no output
        (A, A, None, None, None, None, 1, 100, 100, 0, bf),     # no logits
        (A, A, None, None, None, A, 0, 100, 100, 0, bf),        # no rows
    ]
    for args in bad:
        assert lib.b2_logprobs(*args, None) == B2_ERR_PARAM, args
    assert lib.b2_logprobs_shard(None, None, A, 1, 100, 100, 0, 1, bf, None) == B2_ERR_PARAM
    assert lib.b2_logprobs_shard(A, None, A, 1, 100, 100, 0, 11, bf, None) == B2_ERR_PARAM
    assert lib.b2_logprobs_shard(A, None, A, 1, 100, 99, 0, 1, bf, None) == B2_ERR_PARAM
    assert lib.b2_logprobs_shard(A, None, A, 1, 100, 100, -1, 1, bf, None) == B2_ERR_PARAM
    assert lib.b2_logprobs_shard(A, None, A, 1, 100, 100, 0x7FFFFFFF - 100, 1, bf, None) == B2_ERR_PARAM
    assert lib.b2_logprobs_merge(A, A, None, None, None, 2, 1, 0, None) == B2_ERR_PARAM
    assert lib.b2_logprobs_merge(A, A, None, None, A, 0, 1, 0, None) == B2_ERR_PARAM
    assert lib.b2_logprobs_merge(A, A, None, None, A, 2, 0, 0, None) == B2_ERR_PARAM
    assert lib.b2_logprobs_merge(A, A, None, A, A, 2, 1, 3, None) == B2_ERR_PARAM
    assert lib.b2_logprobs_merge(A, A, None, None, A, 2, 1, 11, None) == B2_ERR_PARAM


def test_decode_stack_rejects_more_than_ten():
    from b200spark import model
    with pytest.raises(AssertionError):
        model.DecodeStack(model.TINY, 1, 16, logprobs=11, device="cpu")


ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "dash-infer_b200", "lib", "libb200spark.so")
CUOBJDUMP = shutil.which("cuobjdump") or next((p for p in ("/usr/local/cuda/bin/cuobjdump",) if os.path.exists(p)), None)


@pytest.mark.skipif(CUOBJDUMP is None, reason="cuobjdump not found")
def test_kernels_have_no_local_memory():
    """the per-thread top-10 stays in registers: no stack frame in any logprobs kernel"""
    out = subprocess.run([CUOBJDUMP, "-res-usage", LIB], check=True, capture_output=True, text=True).stdout
    usage, cur = {}, None
    for line in out.splitlines():
        m = re.match(r"\s*Function (\S+):", line)
        if m:
            cur = m.group(1)
        elif cur is not None and "REG:" in line:
            usage[cur] = int(re.search(r"STACK:(\d+)", line).group(1))
            cur = None
    lp = {k: v for k, v in usage.items() if "logprobs" in k}
    assert len(lp) == 5, sorted(lp)
    assert all(v == 0 for v in lp.values()), lp
