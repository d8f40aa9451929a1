"""Builds libb200shuffle.so in-tree with nvcc for sm_90a (H100; no JIT cache: the .so is loaded from the tree).

    python spark-s3-shuffle_b200/_build.py [--force]
"""
import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "build")
LIB = os.path.join(HERE, "libb200shuffle.so")
HOST_LIB = os.path.join(HERE, "libb200shuffle_host.so")
HOST_SRC = os.path.join(HERE, "host", "shuffle_host.cpp")
SOURCES = ["api.cu", "scan.cu", "partition.cu", "sort.cu", "rows.cu", "rows_hash.cu", "rows_range.cu", "rows_round_robin.cu", "aggregate.cu", "join.cu", "window.cu", "partial_agg.cu", "rows_expand.cu", "exchange.cu", "checksum.cu", "xxh32.cu", "lz4_compress.cu", "lz4_decode.cu", "snappy.cu", "zstd.cu", "zstd_enc.cu", "gen.cu"]
GENCODE = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = GENCODE + [
    "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC,-O2,-Wall",
    "-Xptxas", "-v",
    "--expt-relaxed-constexpr",
]


def _nvcc():
    for cand in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found: libb200shuffle cannot be built (there is no CPU fallback)")


def _deps_mtime():
    m = os.path.getmtime(os.path.abspath(__file__))  # the source list lives here
    for root in (CSRC, os.path.join(HERE, "..", "include")):
        for f in os.listdir(root):
            if f.endswith((".cu", ".cuh", ".h")):
                m = max(m, os.path.getmtime(os.path.join(root, f)))
    return m


def build(force=False, verbose=False):
    if not force and os.path.exists(LIB) and os.path.getmtime(LIB) >= _deps_mtime():
        return LIB
    nvcc = _nvcc()
    os.makedirs(OBJ, exist_ok=True)
    hdr_m = max(os.path.getmtime(os.path.join(CSRC, f)) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h")))
    hdr_m = max(hdr_m, os.path.getmtime(os.path.join(HERE, "..", "include", "b200shuffle.h")))

    def compile_one(src):
        s = os.path.join(CSRC, src)
        o = os.path.join(OBJ, src.replace(".cu", ".o"))
        if not force and os.path.exists(o) and os.path.getmtime(o) >= max(os.path.getmtime(s), hdr_m):
            return o, ""
        cmd = [nvcc] + NVCC_FLAGS + ["-c", s, "-o", o]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed for %s:\n%s\n%s" % (src, r.stdout, r.stderr))
        return o, r.stderr

    with ThreadPoolExecutor(max_workers=len(SOURCES)) as ex:
        results = list(ex.map(compile_one, SOURCES))
    log = "\n".join(r[1] for r in results if r[1])
    with open(os.path.join(OBJ, "ptxas.log"), "a") as f:
        f.write(log)
    if verbose:
        print(log)
    objs = [r[0] for r in results]
    cmd = [nvcc, "-shared", "-o", LIB] + objs + GENCODE + ["-cudart", "static", "-Xcompiler", "-fPIC"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("link failed:\n%s\n%s" % (r.stdout, r.stderr))
    return LIB


def build_host(force=False):
    """libb200shuffle_host.so: the C++ host mirror of the reference's writer/reader/helper classes, linked against
    the C ABI (g++ only; it contains no device code)."""
    lib = build(force=force)
    import glob
    deps = [HOST_SRC, os.path.join(HERE, "..", "include", "b200shuffle_host.h"),
            os.path.join(HERE, "..", "include", "b200shuffle.h"), lib] + glob.glob(os.path.join(HERE, "host", "*.h"))
    if not force and os.path.exists(HOST_LIB) and os.path.getmtime(HOST_LIB) >= max(os.path.getmtime(d) for d in deps):
        return HOST_LIB
    cmd = ["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-pthread", "-o", HOST_LIB, HOST_SRC, "-L" + HERE,
           "-l:libb200shuffle.so", "-Wl,-rpath,$ORIGIN"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("host library build failed:\n%s\n%s" % (r.stdout, r.stderr))
    return HOST_LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
    print(build_host(force="--force" in sys.argv))
