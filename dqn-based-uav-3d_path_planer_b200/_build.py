"""Build libuavrl_b200.so in-tree with nvcc for sm_90a (H100)."""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "build")
LIB = os.path.join(HERE, "libuavrl_b200.so")
SOURCES = ["env.cu", "scenario.cu", "learner.cu", "tc_forward.cu", "tc_train.cu", "train.cu", "eval.cu", "sac.cu", "per.cu", "federate.cu", "replay.cu", "optim.cu"]
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = ARCH + ["-O3", "-lineinfo", "-std=c++17",
                     "-Xcompiler", "-fPIC,-ffp-contract=off", "-Xptxas", "-v"]


def _nvcc():
    for c in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if c and (os.path.isabs(c) and os.path.exists(c) or not os.path.isabs(c)):
            return c
    return "nvcc"


def _deps():
    out = [os.path.join(CSRC, f) for f in os.listdir(CSRC)]
    out.append(os.path.join(HERE, "..", "include", "uavrl.h"))
    out.append(os.path.abspath(__file__))                       # the architecture and compiler flags
    return out


def needs_build():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    return any(os.path.getmtime(p) > t for p in _deps())


def build(force=False, verbose=False):
    """Compile every CUDA source of the hot path for sm_90a and link the C-ABI shared library."""
    srcs = [s for s in SOURCES if os.path.exists(os.path.join(CSRC, s))]
    if not force and not needs_build():
        return LIB
    os.makedirs(OBJ, exist_ok=True)
    nvcc = _nvcc()
    hdr_t = max(os.path.getmtime(p) for p in _deps() if not p.endswith(".cu"))       # headers and the flags in this file

    def one(src):
        obj = os.path.join(OBJ, src.replace(".cu", ".o"))
        sp = os.path.join(CSRC, src)
        if (not force and os.path.exists(obj) and os.path.getmtime(obj) > os.path.getmtime(sp)
                and os.path.getmtime(obj) > hdr_t):
            return obj, ""
        cmd = [nvcc] + NVCC_FLAGS + ["-c", sp, "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed for %s:\n%s\n%s" % (src, r.stdout, r.stderr))
        return obj, r.stderr

    with ThreadPoolExecutor(max_workers=4) as ex:
        res = list(ex.map(one, srcs))
    if verbose:
        for _, log in res:
            sys.stderr.write(log)
    cmd = [nvcc] + ARCH + ["-shared", "-o", LIB] + [o for o, _ in res] + ["-lcudart"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("link failed:\n%s\n%s" % (r.stdout, r.stderr))
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
