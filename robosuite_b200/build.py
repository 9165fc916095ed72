"""In-tree build of libb2s.so (hand-written CUDA for H100, sm_90a; no JIT cache, the .so travels with the tree)."""
import os
import subprocess

_HERE = os.path.dirname(os.path.abspath(__file__))
SO = os.path.join(_HERE, "libb2s.so")
SRC = os.path.join(_HERE, "csrc", "b2s_capi.cu")
# ptxas takes nearly all of the build's time; --split-compile=0 spreads it over every CPU (the same SASS as without it)
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17", "-Xcompiler", "-fPIC",
              "-shared", "-Xptxas", "--split-compile=0"]


def _deps():
    d = [os.path.join(_HERE, "csrc", f) for f in os.listdir(os.path.join(_HERE, "csrc"))]
    d.append(os.path.join(_HERE, "..", "include", "b2s.h"))
    return d


def build(force=False, verbose=False):
    if not force and os.path.exists(SO) and all(os.path.getmtime(p) <= os.path.getmtime(SO) for p in _deps()):
        return SO
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    extra = os.environ.get("B2S_NVCC_EXTRA", "").split()
    out = os.environ.get("B2S_SO_OUT", SO)
    cmd = [nvcc] + NVCC_FLAGS + extra + (["-Xptxas", "-v"] if verbose else []) + ["-o", out, SRC]
    subprocess.check_call(cmd)
    return SO


def build_instr(force=False):
    """-DB2S_INSTR measurement build (device %globaltimer timeline + solver statistics; tools/probe_instr.py, bench.py's
    `roofline.timeline`; the unit queue's stage counters, tools/probe_unit.py).  Never loaded by the product path: selected only
    through B2S_LIB."""
    out = os.path.join(_HERE, "variants", "libb2s_instr.so")
    if not force and os.path.exists(out) and all(os.path.getmtime(p) <= os.path.getmtime(out) for p in _deps()):
        return out
    os.makedirs(os.path.dirname(out), exist_ok=True)
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    subprocess.check_call([nvcc] + NVCC_FLAGS + ["-DB2S_INSTR", "-o", out, SRC])
    return out


if __name__ == "__main__":
    print(build(force=True, verbose=True))
