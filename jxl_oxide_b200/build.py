"""Builds libjxlb200.so (sm_90a, H100) in-tree with nvcc. No JIT cache: the .so travels with the repo snapshot.

Every source is compiled to its own object file under _obj/ (in parallel, only when it or a header changed), then
linked; `python -m jxl_oxide_b200.build --force` rebuilds everything, `-v` adds ptxas resource usage."""
import concurrent.futures
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "_obj")
OUT = os.path.join(HERE, "libjxlb200.so")

SOURCES = [
    "capi.cu", "cuda_backend.cu", "launch_tables.cc", "pipeline.cu",
    "kernels/modular.cu", "kernels/modular_stream.cu", "kernels/entropy.cu", "kernels/blockinfo.cu", "kernels/vardct.cu", "kernels/filters.cu", "kernels/filters_fused.cu", "kernels/jpeg.cu", "kernels/pack.cu",
    "host/entropy.cc", "host/headers.cc", "host/modular_syntax.cc", "host/frame_syntax.cc", "host/planner.cc", "host/icc.cc", "host/jbrd.cc", "host/frame_index.cc",
]

# -fmad=false: the reference's generic float path never contracts a*b+c (SimdVector::muladd is
# mul+add unless built with +fma, crates/jxl-grid/src/simd.rs:177-199); kernels call __fmaf_rn
# exactly where the reference calls mul_add.
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = ["-std=c++17", "-O3"] + ARCH + [
    "-lineinfo", "-fmad=false", "-Xcompiler", "-fPIC,-O2,-ffp-contract=off,-fno-fast-math,-pthread",
]


def _headers_mtime():
    t = os.path.getmtime(os.path.join(os.path.dirname(HERE), "include", "jxlb200.h"))
    for root, _, files in os.walk(CSRC):
        for f in files:
            if f.endswith((".h", ".cuh", ".inc")):
                t = max(t, os.path.getmtime(os.path.join(root, f)))
    return t


def _obj_path(src):
    return os.path.join(OBJ, src.replace("/", "_") + ".o")


def needs_build():
    if not os.path.exists(OUT):
        return True
    t = os.path.getmtime(OUT)
    if _headers_mtime() > t:
        return True
    return any(os.path.exists(os.path.join(CSRC, s)) and os.path.getmtime(os.path.join(CSRC, s)) > t for s in SOURCES)


def build(force=False, verbose=False):
    if not force and not needs_build():
        return OUT
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    os.makedirs(OBJ, exist_ok=True)
    hdr_t = _headers_mtime()
    srcs = [s for s in SOURCES if os.path.exists(os.path.join(CSRC, s))]

    def compile_one(src):
        obj = _obj_path(src)
        path = os.path.join(CSRC, src)
        if not force and os.path.exists(obj) and os.path.getmtime(obj) > max(os.path.getmtime(path), hdr_t):
            return obj
        cmd = [nvcc] + NVCC_FLAGS + (["-Xptxas=-v"] if verbose else []) + ["-x", "cu", "-c", path, "-o", obj]
        subprocess.check_call(cmd, cwd=CSRC)
        return obj
    with concurrent.futures.ThreadPoolExecutor(max_workers=min(8, os.cpu_count() or 1)) as ex:
        objs = list(ex.map(compile_one, srcs))
    subprocess.check_call([nvcc, "--shared"] + ARCH + ["-Xcompiler", "-fPIC,-pthread"] + objs +
                          ["-o", OUT, "-lcudart", "-ldl"], cwd=CSRC)
    return OUT


if __name__ == "__main__":
    build(force="--force" in sys.argv, verbose="-v" in sys.argv)
    print(OUT)
