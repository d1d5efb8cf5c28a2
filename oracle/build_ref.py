"""TEST / TOOLING INFRASTRUCTURE (oracle/): builds oracle/_ref/ from the reference's own sources in a checkout of the upstream
Hetu-Galvatron tree (never copied into the repo; oracle/_ref/ is git-ignored).

The hot path of the reference is Python over torch/NCCL -- there is no C/C++ source OF THE PATH to compile (DESIGN.md section 5).
The one C++ file the reference ships is the Search Engine's dynamic-programming core, csrc/dp_core.cpp (pybind11); it is what
`scripts/search_strategy.py` runs, unmodified, to search strategies from measured profiles, so it is built here.
Called by scripts/search_strategy.py with the checkout's path; a no-op when the source is absent."""
import os
import subprocess
import sys
import sysconfig

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def build(ref):
    src = os.path.join(ref, "csrc", "dp_core.cpp")
    if not os.path.exists(src):
        print("[oracle/build_ref] %s not present: nothing to build" % src)
        return None
    out_dir = os.path.join(ROOT, "oracle", "_ref")
    os.makedirs(out_dir, exist_ok=True)
    so = os.path.join(out_dir, "galvatron_dp_core" + sysconfig.get_config_var("EXT_SUFFIX"))
    if os.path.exists(so) and os.path.getmtime(so) >= os.path.getmtime(src):
        return so
    inc = subprocess.check_output([sys.executable, "-m", "pybind11", "--includes"], text=True).split()
    cmd = ["g++", "-O3", "-shared", "-std=c++17", "-fPIC", *inc, src, "-o", so]
    print(" ".join(cmd), flush=True)
    subprocess.check_call(cmd)
    return so


if __name__ == "__main__":
    build(sys.argv[1])
