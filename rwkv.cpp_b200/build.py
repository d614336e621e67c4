"""Builds rwkv.cpp_b200/librwkv.so (the C-ABI library) in-tree with nvcc for sm_90a.

    python rwkv.cpp_b200/build.py [--force]

The .so is git-ignored. nvcc cross-compiles without a GPU.
"""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "build")
LIB = os.path.join(HERE, "librwkv.so")

SOURCES = [
    "api.cpp", "adapter.cpp", "ggml_file.cpp", "quantizer.cpp", "model.cu", "engine.cu",
    "kernels/gemv.cu", "kernels/gemv_tma.cu", "kernels/gemv_kquant.cu", "kernels/gemm_tc.cu", "kernels/pipe.cu", "kernels/glue.cu", "kernels/wkv.cu", "kernels/sampling.cu", "kernels/columns.cu",
    "kernels/score.cu", "kernels/lora.cu",
]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
COMMON = ["-std=c++17", "-O3", "-lineinfo", "-diag-suppress", "1675", "-DRWKV_SHARED", "-DRWKV_BUILD",
          "-Xcompiler", "-fPIC,-fvisibility=hidden,-ffp-contract=off,-Wall,-Wno-unused-function,-Wno-unknown-pragmas", "-Xptxas", "-v" if os.environ.get("RWKV_PTXAS_V") else "-O3"]


def _headers_mtime():
    newest = 0.0
    for root, _, files in os.walk(CSRC):
        for f in files:
            if f.endswith((".h", ".cuh")):
                newest = max(newest, os.path.getmtime(os.path.join(root, f)))
    inc = os.path.join(HERE, "..", "include")
    for f in os.listdir(inc):
        newest = max(newest, os.path.getmtime(os.path.join(inc, f)))
    return newest


def _compile(src, force, hdr_mtime):
    path = os.path.join(CSRC, src)
    obj = os.path.join(OBJ, src.replace("/", "_") + ".o")
    if not force and os.path.exists(obj) and os.path.getmtime(obj) >= max(os.path.getmtime(path), hdr_mtime):
        return obj, None
    cmd = [NVCC] + ARCH + COMMON + ["-x", "cu", "-c", path, "-o", obj]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("nvcc failed for %s:\n%s\n%s" % (src, r.stdout, r.stderr))
    return obj, (r.stdout + r.stderr).strip()


def build(force=False, verbose=False):
    os.makedirs(OBJ, exist_ok=True)
    hdr = _headers_mtime()
    with ThreadPoolExecutor(max_workers=min(8, len(SOURCES))) as ex:
        results = list(ex.map(lambda s: _compile(s, force, hdr), SOURCES))
    objs = [o for o, _ in results]
    rebuilt = [log for _, log in results if log is not None]
    if verbose:
        for log in rebuilt:
            if log:
                print(log)
    if rebuilt or not os.path.exists(LIB) or any(os.path.getmtime(o) > os.path.getmtime(LIB) for o in objs):
        cmd = [NVCC] + ARCH + ["-shared", "-o", LIB] + objs + ["-Xlinker", "--no-undefined"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("link failed:\n%s\n%s" % (r.stdout, r.stderr))
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
