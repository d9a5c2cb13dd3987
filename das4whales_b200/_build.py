"""Build libd4w.so (all CUDA kernels + the C ABI) for the H100 (sm_90a), in-tree, with nvcc.

`nvcc` cross-compiles without a GPU, so the library can be built on a machine without one and
copied with the source tree to the GPU machine.
"""
import os
import shutil
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libd4w.so")
SOURCES = ["d4w_fk.cu", "d4w_rows.cu", "d4w_xcorr_same.cu", "d4w_image.cu", "d4w_noise.cu"]
GENCODE = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = ["-std=c++17", "-O3", "--expt-relaxed-constexpr"] + GENCODE + [
              "-lineinfo", "-Xcompiler", "-fPIC", "-Wno-deprecated-gpu-targets"]


def _nvcc():
    exe = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(exe):
        raise RuntimeError("nvcc not found: cannot build das4whales_b200/libd4w.so")
    return exe


def _stale():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    # this file too: a library built with other flags (another architecture) is stale
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(HERE, "..", "include", "d4w.h"), __file__]
    return any(os.path.getmtime(d) > t for d in deps if os.path.exists(d))


def _sync_header():
    """Keep the in-package copy of the C header identical to include/d4w.h."""
    src, dst = os.path.join(HERE, "..", "include", "d4w.h"), os.path.join(HERE, "d4w.h")
    if os.path.exists(src):
        with open(src, "rb") as f:
            text = f.read()
        if not os.path.exists(dst) or open(dst, "rb").read() != text:
            with open(dst, "wb") as f:
                f.write(text)


def build_library(force=False, verbose=False):
    """Compile every .cu into one shared library. Returns the path of libd4w.so."""
    _sync_header()
    if not force and not _stale():
        return LIB
    srcs = [os.path.join(CSRC, s) for s in SOURCES if os.path.exists(os.path.join(CSRC, s))]
    objs = []
    procs = []
    for s in srcs:
        o = os.path.splitext(s)[0] + ".o"
        objs.append(o)
        cmd = [_nvcc()] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-c", s, "-o", o]
        procs.append((cmd, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    for cmd, p in procs:
        out, _ = p.communicate()
        if verbose and out:
            print(out)
        if p.returncode != 0:
            raise RuntimeError("nvcc failed: " + " ".join(cmd) + "\n" + (out or ""))
    cmd = [_nvcc(), "-shared"] + GENCODE + ["-o", LIB] + objs + ["-lcudart"]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        raise RuntimeError("link failed: " + " ".join(cmd) + "\n" + r.stdout)
    return LIB


if __name__ == "__main__":
    import sys
    print(build_library(force=True, verbose="-v" in sys.argv))
