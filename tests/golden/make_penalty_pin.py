"""Generate tests/golden/penalty_pin.npz: what the reference's own logits processor (allspark::cuda::LogitsProcessor,
beam_search.cu) computes on the inputs of tests/test_penalty_gpu.py::test_matches_restatement.

Two steps, because the reference checkout and the GPU need not be on the same machine:
    python tests/golden/make_penalty_pin.py --build [REFERENCE_DIR]   # nvcc, no GPU: beam_search.cu + a C shim
    python tests/golden/make_penalty_pin.py                           # on a GPU: run it, write the .npz
--build compiles the reference's unmodified beam_search.cu with the flags of oracle/build_ref.py (sm_90, -O2,
--use_fast_math) into tests/golden/_penalty_ref/libpenalty_ref.so (git-ignored).  The stub headers it needs (a null
glog LOG, the BatchGencfg field layout, an opaque hiednn handle) and the shim are written next to it from the strings
below; nothing of the reference is stored in the repository.

Stored per case "{ft}_{n}_{rows}" (penalty_ref.CASES; the inputs are regenerated from penalty_ref.case's seeds):
  {case}_idx    uint32: the flat positions r * n + c where the reference's output bits differ from the input's, delta
                encoded (the first entry is the position itself)
  {case}_bits   uint16: the reference's output bits at those positions
  {case}_crc    crc32 of the input logits' bits (a generator drift check)
The reference writes out of bounds for an eos id < 0 while cur_len < min_length; those rows get min_length 0, which is
what eos id < 0 means to b2_penalize.
"""
import ctypes as C
import os
import subprocess
import sys
import zlib

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
OUT = os.path.join(HERE, "_penalty_ref")
SO = os.path.join(OUT, "libpenalty_ref.so")
sys.path.insert(0, os.path.dirname(HERE))

STUBS = {
    "glog/logging.h": """#pragma once
#include <ostream>
#include <sstream>
namespace penalty_pin { struct NullLog { template <class T> NullLog& operator<<(const T&) { return *this; }
  NullLog& operator<<(std::ostream& (*)(std::ostream&)) { return *this; } }; }
#define LOG(x) penalty_pin::NullLog()
#define DLOG(x) penalty_pin::NullLog()
""",
    "common.h": """#pragma once
namespace allspark {
struct BatchGencfg {
  int batch_size = 0;
  void* repetition_penalty_list = nullptr;
  void* presence_penalty_list = nullptr;
  void* frequency_penalty_list = nullptr;
  void* no_repeat_ngram_size_list = nullptr;
  void* min_length_list = nullptr;
  void* eos_token_id_list = nullptr;
  void* cur_len_list = nullptr;
  void* input_len_list = nullptr;
  void* suppress_repetition_in_generation_list = nullptr;
};
}  // namespace allspark
""",
    "hiednn_cuda.h": "#pragma once\ntypedef struct hiednnCudaContext* hiednnCudaHandle_t;\n",
}

SHIM = r"""
#include "cuda_common.h"
#include "cuda_kernel.h"
extern "C" int penalty_ref_run(void* score, const int64_t* in_ids, int batch, int max_len, int vocab, void* rep,
                               void* pres, void* freq, void* ngram, void* min_len, void* eos, void* cur_len,
                               void* input_len, void* suppress, void* ws, size_t ws_bytes, int fp16, void* stream) {
  allspark::BatchGencfg g;
  g.batch_size = batch;
  g.repetition_penalty_list = rep;
  g.presence_penalty_list = pres;
  g.frequency_penalty_list = freq;
  g.no_repeat_ngram_size_list = ngram;
  g.min_length_list = min_len;
  g.eos_token_id_list = eos;
  g.cur_len_list = cur_len;
  g.input_len_list = input_len;
  g.suppress_repetition_in_generation_list = suppress;
  if (fp16)
    allspark::cuda::LogitsProcessor<half>((half*)score, in_ids, batch, max_len, vocab, g, ws, ws_bytes, (cudaStream_t)stream);
  else
    allspark::cuda::LogitsProcessor<hie::bfloat16>((hie::bfloat16*)score, in_ids, batch, max_len, vocab, g, ws, ws_bytes,
                                                   (cudaStream_t)stream);
  return (int)cudaGetLastError();
}
"""


def build(ref):
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    stubs = os.path.join(OUT, "stubs")
    for name, text in STUBS.items():
        os.makedirs(os.path.dirname(os.path.join(stubs, name)), exist_ok=True)
        with open(os.path.join(stubs, name), "w") as f:
            f.write(text)
    shim = os.path.join(OUT, "shim.cu")
    with open(shim, "w") as f:
        f.write(SHIM)
    kern = os.path.join(ref, "csrc", "core", "kernel")
    inc = ["-I", stubs, "-I", os.path.join(kern, "cuda"), "-I", os.path.join(ref, "csrc", "common"), "-I", kern,
           "-I", os.path.join(ref, "csrc", "device"), "-I", os.path.join(ref, "csrc")]
    flags = ["-gencode", "arch=compute_90,code=sm_90", "-std=c++17", "-O2", "-DNDEBUG", "-DENABLE_BF16", "-DENABLE_FP16",
             "-DENABLE_CUDA", "--expt-relaxed-constexpr", "--extended-lambda", "--use_fast_math", "-Xcompiler", "-fPIC",
             "-x", "cu", "-w"]
    objs = []
    for src in (os.path.join(kern, "cuda", "beam_search.cu"), shim):
        obj = os.path.join(OUT, os.path.basename(src) + ".o")
        subprocess.run([nvcc] + flags + inc + ["-c", src, "-o", obj], check=True)
        objs.append(obj)
    subprocess.run([nvcc, "-gencode", "arch=compute_90,code=sm_90", "-shared", "-o", SO] + objs, check=True)
    return SO


def input_bits(x, ft):
    import penalty_ref as P
    return P.bits(x, ft)


def run_case(lib, ft, n, rows):
    import torch

    import penalty_ref as P
    hists, prompts, prm, x = P.case(ft, n, rows)
    max_len = 256
    dev = "cuda"
    tok = torch.zeros(rows, max_len, dtype=torch.int64)
    for r, h in enumerate(hists):
        tok[r, :len(h)] = torch.as_tensor(h, dtype=torch.int64)
    minl = [m if e >= 0 else 0 for m, e in zip(prm["min_length"], prm["eos_id"])]
    f32 = lambda v: torch.tensor(v, dtype=torch.float32, device=dev)
    i32 = lambda v: torch.tensor([int(a) for a in v], dtype=torch.int32, device=dev)
    args = [f32(prm["repetition"]), f32(prm["presence"]), f32(prm["frequency"]), i32(prm["no_repeat_ngram"]), i32(minl),
            i32(prm["eos_id"]), i32([len(h) for h in hists]), i32(prompts), i32(prm["suppress"])]
    bits_in = input_bits(x, ft)
    score = torch.from_numpy(bits_in.view(np.int16).copy()).to(dev)
    ids = tok.to(dev)
    ws = torch.empty(rows * n * 4, dtype=torch.uint8, device=dev)
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    e = lib.penalty_ref_run(C.c_void_p(score.data_ptr()), C.c_void_p(ids.data_ptr()), rows, max_len, n,
                            *[C.c_void_p(a.data_ptr()) for a in args], C.c_void_p(ws.data_ptr()), C.c_size_t(ws.numel()),
                            int(ft == "fp16"), st)
    torch.cuda.synchronize()
    assert e == 0, e
    out = score.cpu().numpy().view(np.uint16)
    pos = np.flatnonzero(out.reshape(-1) != bits_in.reshape(-1)).astype(np.uint32)
    idx = np.diff(pos, prepend=np.uint32(0)).astype(np.uint32)
    return idx, out.reshape(-1)[pos], zlib.crc32(bits_in.tobytes())


def main():
    if "--build" in sys.argv:
        rest = [a for a in sys.argv[1:] if a != "--build"]
        print("built:", build(rest[0] if rest else os.environ.get("B2_REFERENCE", "/root/reference")))
        return
    import penalty_ref as P
    lib = C.CDLL(SO)
    lib.penalty_ref_run.restype = C.c_int
    store = {}
    for ft, n, rows in P.CASES:
        idx, bits, crc = run_case(lib, ft, n, rows)
        key = "%s_%d_%d" % (ft, n, rows)
        store[key + "_idx"], store[key + "_bits"] = idx, bits
        store[key + "_crc"] = np.uint32(crc)
        print(key, "changed", idx.size, flush=True)
    out = sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "penalty_pin.npz")
    np.savez_compressed(out, **store)
    print("wrote", out)


if __name__ == "__main__":
    main()
