"""ctypes binding of include/b200spark.h.  There is NO fallback: if the native library is missing the
import fails loudly (build it with `python dash-infer_b200/build.py`)."""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_DIR = os.path.normpath(os.path.join(_HERE, "..", "..", "lib"))
LIB_PATH = os.path.join(LIB_DIR, "libb200spark.so")

# every symbol include/b200spark.h declares (checked by tests/test_abi.py)
SYMBOLS = [
    "b2_status_string", "b2_last_error", "b2_version", "b2_set_pdl",
    "b2_gemm_wq_create", "b2_gemm_wq_destroy", "b2_gemm_wq_packed_bytes", "b2_gemm_wq_prepare_weights",
    "b2_gemm_wq_prepare_swiglu", "b2_gemm_wq_attach_packed", "b2_gemm_wq_workspace_bytes", "b2_gemm_wq_run", "b2_gemm_wq_run_fused", "b2_gemm_wq_sumsq_parts",
    "b2_gemm_wq_algo_bytes", "b2_quant_fp8", "b2_gemm_wq_run_fp8",
    "b2_span_bytes", "b2_span_cache_append", "b2_span_context_copy", "b2_span_attn_create", "b2_span_attn_destroy",
    "b2_span_attn_workspace_bytes", "b2_span_attn_run", "b2_span_attn_algo_bytes",
    "b2_span_cache_append_tokens", "b2_span_attn_tokens_workspace_bytes", "b2_span_attn_run_tokens", "b2_spec_accept",
    "b2_span_cache_append_tree", "b2_span_attn_run_tree", "b2_spec_accept_tree", "b2_span_cache_compact",
    "b2_rmsnorm", "b2_rotary", "b2_binary", "b2_embedding", "b2_argmax", "b2_argmax_shard", "b2_argmax_merge", "b2_lens_add",
    "b2_rmsnorm_ft", "b2_binary_ft", "b2_argmax_ft",
    "b2_comm_create", "b2_comm_destroy", "b2_comm_buffer_bytes", "b2_comm_export", "b2_comm_connect", "b2_comm_connect_pointers",
    "b2_comm_local_buffer", "b2_comm_error", "b2_allreduce", "b2_allgather", "b2_gemm_wq_run_allreduce",
]


class GemmDesc(C.Structure):
    _fields_ = [("K", C.c_int32), ("N", C.c_int32), ("wbits", C.c_int32), ("group_size", C.c_int32),
                ("ft", C.c_int32), ("qtype", C.c_int32), ("max_m", C.c_int32), ("reserved", C.c_int32)]


class SpanCfg(C.Structure):
    _fields_ = [("ft", C.c_int32), ("quant_mode", C.c_int32), ("n_heads", C.c_int32), ("n_groups", C.c_int32),
                ("head_size", C.c_int32), ("span_len", C.c_int32), ("max_spans_per_seq", C.c_int32),
                ("reserved", C.c_int32)]


class GemmFuse(C.Structure):
    _fields_ = [("norm_sumsq", C.c_void_p), ("norm_gamma", C.c_void_p), ("norm_parts", C.c_int32), ("norm_hidden", C.c_int32),
                ("norm_eps", C.c_float), ("reserved", C.c_int32), ("sumsq_out", C.c_void_p),
                ("xg_out", C.c_void_p), ("gamma_out", C.c_void_p), ("ldxg", C.c_int64)]


class RopeCfg(C.Structure):
    _fields_ = [("base", C.c_float), ("rotary_dim", C.c_int32), ("reserved", C.c_int32)]


DT_F32, DT_F16, DT_I8, DT_BF16, DT_U8 = 1, 2, 3, 9, 10
ACT_NONE, ACT_TANH, ACT_GELU_ERF, ACT_GELU_TANH, ACT_RELU, ACT_SILU, ACT_SIGMOID = range(7)
ACT_SWIGLU = 100
BIN_ADD, BIN_MUL = 1, 2
KV_NONE, KV_I8, KV_U4 = 0, 1, 2
KV_FP8 = 3  # extension (not a span::QuantMode value): fp8-e4m3 KV cache, head 128 only
COMM_HANDLE_BYTES = 64


class B2Error(RuntimeError):
    pass


def _load():
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"b200spark native library not found at {LIB_PATH}; build it first: python dash-infer_b200/build.py "
            "(there is no CPU/PyTorch fallback for the hot path)")
    lib = C.CDLL(LIB_PATH, mode=C.RTLD_GLOBAL)
    vp, i32, i64, sz, f32 = C.c_void_p, C.c_int, C.c_int64, C.c_size_t, C.c_float
    sig = {
        "b2_status_string": (C.c_char_p, [i32]),
        "b2_last_error": (C.c_char_p, []),
        "b2_version": (C.c_char_p, []),
        "b2_set_pdl": (None, [i32]),
        "b2_gemm_wq_create": (i32, [C.POINTER(vp), C.POINTER(GemmDesc)]),
        "b2_gemm_wq_destroy": (i32, [vp]),
        "b2_gemm_wq_packed_bytes": (sz, [vp]),
        "b2_gemm_wq_prepare_weights": (i32, [vp, vp, vp, vp, vp, vp]),
        "b2_gemm_wq_prepare_swiglu": (i32, [vp, vp, vp, vp, vp, vp, vp, vp]),
        "b2_gemm_wq_attach_packed": (i32, [vp, vp, vp, vp]),
        "b2_gemm_wq_workspace_bytes": (sz, [vp, i32]),
        "b2_gemm_wq_run": (i32, [vp, vp, i64, vp, i64, i32, vp, vp, i32, f32, vp, sz, vp]),
        "b2_gemm_wq_run_fused": (i32, [vp, vp, i64, vp, i64, i32, vp, vp, i32, f32, vp, sz, C.POINTER(GemmFuse), vp]),
        "b2_gemm_wq_sumsq_parts": (i32, [vp]),
        "b2_gemm_wq_algo_bytes": (sz, [vp, i32]),
        "b2_quant_fp8": (i32, [vp, i64, vp, vp, vp, vp, i32, i32, f32, vp]),
        "b2_gemm_wq_run_fp8": (i32, [vp, vp, i64, vp, vp, vp, i64, i32, vp, vp, i32, f32, vp, sz, vp]),
        "b2_span_bytes": (sz, [C.POINTER(SpanCfg)]),
        "b2_span_cache_append": (i32, [C.POINTER(SpanCfg), vp, vp, vp, vp, vp, i32, C.POINTER(RopeCfg), vp]),
        "b2_span_context_copy": (i32, [C.POINTER(SpanCfg), vp, vp, i64, i32, vp]),
        "b2_span_attn_create": (i32, [C.POINTER(vp), C.POINTER(SpanCfg), i32]),
        "b2_span_attn_destroy": (i32, [vp]),
        "b2_span_attn_workspace_bytes": (sz, [vp, i32, i32]),
        "b2_span_attn_run": (i32, [vp, vp, vp, vp, vp, vp, i32, i32, vp, sz, f32, vp]),
        "b2_span_attn_algo_bytes": (sz, [C.POINTER(SpanCfg), i64]),
        "b2_span_cache_append_tokens": (i32, [C.POINTER(SpanCfg), vp, vp, vp, vp, vp, i32, i32, C.POINTER(RopeCfg), vp]),
        "b2_span_attn_tokens_workspace_bytes": (sz, [vp, i32, i32, i32]),
        "b2_span_attn_run_tokens": (i32, [vp, vp, vp, vp, vp, vp, i32, i32, i32, vp, sz, f32, vp]),
        "b2_spec_accept": (i32, [vp, vp, vp, vp, vp, vp, i32, i32, vp]),
        "b2_span_cache_append_tree": (i32, [C.POINTER(SpanCfg), vp, vp, vp, vp, vp, vp, i32, i32, C.POINTER(RopeCfg), vp]),
        "b2_span_attn_run_tree": (i32, [vp, vp, vp, vp, vp, vp, vp, i32, i32, i32, vp, sz, f32, vp]),
        "b2_spec_accept_tree": (i32, [vp, vp, vp, vp, vp, vp, vp, vp, i32, i32, vp]),
        "b2_span_cache_compact": (i32, [C.POINTER(SpanCfg), vp, vp, i32, vp, vp, vp, i32, i32, vp]),
        "b2_rmsnorm": (i32, [vp, vp, vp, i32, i32, f32, vp]),
        "b2_rmsnorm_ft": (i32, [vp, vp, vp, i32, i32, f32, i32, vp]),
        "b2_binary_ft": (i32, [vp, vp, vp, i64, i32, i32, vp]),
        "b2_argmax_ft": (i32, [vp, vp, vp, i32, i32, i64, i64, i32, vp]),
        "b2_rotary": (i32, [vp, vp, i32, i32, i32, i32, C.POINTER(RopeCfg), vp]),
        "b2_binary": (i32, [vp, vp, vp, i64, i32, vp]),
        "b2_embedding": (i32, [vp, vp, vp, i32, i32, vp]),
        "b2_argmax": (i32, [vp, vp, i32, i32, i64, vp]),
        "b2_argmax_shard": (i32, [vp, vp, vp, i32, i32, i64, i64, vp]),
        "b2_lens_add": (i32, [vp, i32, i32, vp]),
        "b2_argmax_merge": (i32, [vp, vp, vp, i32, i32, vp]),
        "b2_comm_create": (i32, [C.POINTER(vp), i32, i32, sz]),
        "b2_comm_destroy": (i32, [vp]),
        "b2_comm_buffer_bytes": (sz, [i32, sz]),
        "b2_comm_export": (i32, [vp, vp]),
        "b2_comm_connect": (i32, [vp, vp]),
        "b2_comm_connect_pointers": (i32, [vp, vp]),
        "b2_comm_local_buffer": (vp, [vp]),
        "b2_comm_error": (i32, [vp]),
        "b2_allreduce": (i32, [vp, vp, vp, vp, i64, i32, vp]),
        "b2_allgather": (i32, [vp, vp, vp, i32, vp]),
        "b2_gemm_wq_run_allreduce": (i32, [vp, vp, i64, vp, i64, i32, vp, vp, f32, vp, sz, vp, vp]),
    }
    for name, (res, args) in sig.items():
        fn = getattr(lib, name)  # AttributeError here == ABI drift: fail loudly
        fn.restype = res
        fn.argtypes = args
    return lib


lib = _load()
if os.environ.get("B2_PDL", "1") == "0":
    lib.b2_set_pdl(0)


def check(status, what=""):
    if status != 0:
        raise B2Error(f"{what}: {lib.b2_status_string(status).decode()} ({lib.b2_last_error().decode()})")
