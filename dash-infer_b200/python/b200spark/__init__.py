"""b200spark — H100-native quantized decode hot path behind DashInfer's operator API (Python front end).

The native library is mandatory: importing this package without `dash-infer_b200/lib/libb200spark.so`
raises ImportError (no CPU / eager-PyTorch fallback exists on the product path).
"""
from . import _lib  # noqa: F401  (fails loudly if the .so is missing)
from ._lib import (ACT_GELU_ERF, ACT_GELU_TANH, ACT_NONE, ACT_RELU, ACT_SIGMOID, ACT_SILU, ACT_SWIGLU, ACT_TANH, BIN_ADD,  # noqa: F401
                   BIN_MUL, KV_I8, KV_NONE, KV_U4, B2Error, lib)
from . import quantize  # noqa: F401

__all__ = ["lib", "quantize"]
