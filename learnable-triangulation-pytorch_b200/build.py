"""Build liblt_b200.so (all CUDA kernels + the C ABI of include/lt_b200.h) for sm_90a (H100), in-tree.

nvcc cross-compiles without a GPU.  The .so, its object files and the source-digest stamp are build
products (git-ignored).  `python -m`-free usage: `from lt_b200 import build; build.build()`.
"""
import hashlib
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "liblt_b200.so")
STAMP = os.path.join(HERE, ".liblt_b200.stamp")
SOURCES = ["capi.cu", "unproject.cu", "softargmax.cu", "conv_simt.cu", "conv_tc.cu", "conv_tail.cu", "misc.cu", "algebraic.cu", "backward.cu"]
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = ARCH + ["-O3", "-lineinfo", "-std=c++17",
                     "--expt-relaxed-constexpr", "-Xcompiler", "-fPIC", "-Xptxas", "-v"]


def _digest():
    h = hashlib.sha256()
    names = sorted(os.listdir(CSRC)) + ["../../include/lt_b200.h"]
    for name in names:
        path = os.path.join(CSRC, name)
        if os.path.isfile(path):
            with open(path, "rb") as f:
                h.update(name.encode())
                h.update(f.read())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def is_current():
    if not (os.path.exists(LIB) and os.path.exists(STAMP)):
        return False
    with open(STAMP) as f:
        return f.read().strip() == _digest()


def build(force=False, verbose=False):
    """Compile every .cu under csrc/ into liblt_b200.so. Returns the library path."""
    if not force and is_current():
        return LIB
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    objs = []
    procs = []
    os.makedirs(os.path.join(HERE, "build"), exist_ok=True)
    for src in SOURCES:
        obj = os.path.join(HERE, "build", src.replace(".cu", ".o"))
        cmd = [nvcc] + NVCC_FLAGS + ["-c", os.path.join(CSRC, src), "-o", obj]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(obj)
    log = []
    failed = False
    for src, pr in procs:
        out, _ = pr.communicate()
        log.append("== %s ==\n%s" % (src, out))
        failed |= pr.returncode != 0
    with open(os.path.join(HERE, "build", "nvcc.log"), "w") as f:
        f.write("\n".join(log))
    if failed:
        sys.stderr.write("\n".join(log))
        raise RuntimeError("nvcc failed (see build/nvcc.log)")
    link = [nvcc, "-shared", "-o", LIB] + objs + ARCH
    res = subprocess.run(link, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if res.returncode != 0:
        sys.stderr.write(res.stdout)
        raise RuntimeError("link failed")
    with open(STAMP, "w") as f:
        f.write(_digest())
    if verbose:
        print("\n".join(log))
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
