"""Build the in-tree native libraries for sm_90a (H100) with nvcc (no GPU needed to compile).

  lib/libb200spark.so      CUDA kernels + the C ABI of include/b200spark.h   (csrc/*.cu)
  lib/liballspark_b200.so  allspark-shaped C++ operator layer over the C ABI  (host/*.cpp), if present

Usage: python dash-infer_b200/build.py [--force] [--verbose]
"""
import hashlib
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
LIB = os.path.join(HERE, "lib")
OBJ = os.path.join(HERE, "build")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
CUFLAGS = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr",
           "-Xptxas", "-v" if os.environ.get("B2_PTXAS_V") else "-warn-spills"] + os.environ.get("B2_EXTRA_NVCC", "").split()


def _stamp(path, extra=""):
    h = hashlib.sha1()
    with open(path, "rb") as f:
        h.update(f.read())
    for dep in sorted(os.listdir(os.path.dirname(path))):
        if dep.endswith((".cuh", ".h", ".hpp")):
            with open(os.path.join(os.path.dirname(path), dep), "rb") as f:
                h.update(f.read())
    with open(os.path.join(ROOT, "include", "b200spark.h"), "rb") as f:
        h.update(f.read())
    h.update(extra.encode())
    return h.hexdigest()


def _run(cmd, verbose):
    if verbose:
        print(" ".join(cmd), flush=True)
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0 or verbose or os.environ.get("B2_PTXAS_V"):
        sys.stdout.write(r.stdout)
    if r.returncode != 0:
        raise RuntimeError("build failed: " + " ".join(cmd))


def _compile_all(srcs, flags, compiler_cmd, tag, force, verbose):
    os.makedirs(OBJ, exist_ok=True)
    objs, jobs = [], []
    for src in srcs:
        obj = os.path.join(OBJ, tag + "_" + os.path.basename(src) + ".o")
        stamp_file = obj + ".stamp"
        stamp = _stamp(src, " ".join(flags))
        objs.append(obj)
        if not force and os.path.exists(obj) and os.path.exists(stamp_file) and open(stamp_file).read() == stamp:
            continue
        jobs.append((compiler_cmd + flags + ["-c", src, "-o", obj], stamp_file, stamp))
    def work(job):
        cmd, stamp_file, stamp = job
        _run(cmd, verbose)
        with open(stamp_file, "w") as f:
            f.write(stamp)
    with ThreadPoolExecutor(max_workers=min(8, max(1, len(jobs)))) as ex:
        list(ex.map(work, jobs))
    return objs, bool(jobs)


def build(force=False, verbose=False):
    os.makedirs(LIB, exist_ok=True)
    csrc = os.path.join(HERE, "csrc")
    cu = sorted(os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith(".cu"))
    objs, changed = _compile_all(cu, ARCH + CUFLAGS, [NVCC], "cu", force, verbose)
    so = os.path.join(LIB, "libb200spark.so")
    if changed or not os.path.exists(so):
        _run([NVCC] + ARCH + ["-shared", "-o", so] + objs, verbose)
    out = [so]
    host = os.path.join(HERE, "host")
    cpp = sorted(os.path.join(host, f) for f in os.listdir(host) if f.endswith(".cpp")) if os.path.isdir(host) else []
    if cpp:
        flags = ["-O2", "-std=c++17", "-Xcompiler", "-fPIC", "-I", os.path.join(ROOT, "include"), "-I", host]
        hobjs, hchanged = _compile_all(cpp, flags, [NVCC, "-x", "cu"] + ARCH, "host", force, verbose)
        hso = os.path.join(LIB, "liballspark_b200.so")
        if hchanged or changed or not os.path.exists(hso):
            _run([NVCC] + ARCH + ["-shared", "-o", hso] + hobjs + ["-L", LIB, "-lb200spark", "-Xlinker", "-rpath=$ORIGIN"], verbose)
        out.append(hso)
    return out


if __name__ == "__main__":
    libs = build(force="--force" in sys.argv, verbose="--verbose" in sys.argv)
    print("built:", *libs)
