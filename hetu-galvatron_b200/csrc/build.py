"""Build libbg_galvatron.so in-tree for sm_90a (nvcc cross-compiles without a GPU).

    python hetu-galvatron_b200/csrc/build.py [--force]

The .so and the object files are build products (git-ignored); rebuilt whenever a source or header is newer.
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
SOURCES = ["bg_comm.cu", "bg_coll.cu", "bg_ops.cu", "bg_gemm.cu"]
HEADERS = ["bg_common.cuh", "bg_ctx.cuh", os.path.join(ROOT, "include", "bg_galvatron.h")]
LIB = os.path.join(HERE, "libbg_galvatron.so")
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17", "-Xcompiler", "-fPIC",
              "-I" + os.path.join(ROOT, "include")]


def _nvcc():
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    return "nvcc"


def _stale():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(HERE, s) for s in SOURCES] + [h if os.path.isabs(h) else os.path.join(HERE, h) for h in HEADERS]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=True):
    if not force and not _stale():
        return LIB
    objs = []
    procs = []
    for src in SOURCES:
        obj = os.path.join(HERE, src.replace(".cu", ".o"))
        objs.append(obj)
        cmd = [_nvcc()] + NVCC_FLAGS + ["-c", os.path.join(HERE, src), "-o", obj]
        if verbose:
            print(" ".join(cmd), flush=True)
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            raise RuntimeError("nvcc failed on %s:\n%s" % (src, out))
        if verbose and out.strip():
            print(out)
    cmd = [_nvcc(), "-shared", "-o", LIB] + objs + ["-gencode", "arch=compute_90a,code=sm_90a"]
    if verbose:
        print(" ".join(cmd), flush=True)
    subprocess.run(cmd, check=True)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv))
