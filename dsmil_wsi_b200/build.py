"""Builds libdsmil_b200.so in-tree with nvcc for sm_90a (no JIT cache: the .so is built next to the sources).

    python -m dsmil_wsi_b200.build          # or: from dsmil_wsi_b200.build import build_library
"""
import hashlib
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.path.join(HERE, "lib")
LIB = os.path.join(LIBDIR, "libdsmil_b200.so")
SOURCES = ["abi.cu"]
HOST_CSRC = os.path.join(HERE, "csrc_host")
HOST_LIB = os.path.join(LIBDIR, "libdsmil_host.so")
HOST_SOURCES = ["bagcsv.c", "jpegparse.c"]
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]


def _nvcc():
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found (set NVCC=/path/to/nvcc)")


def _digest():
    h = hashlib.sha256()
    files = sorted(os.listdir(CSRC)) + [os.path.join("..", "..", "include", "dsmil_b200.h")]
    for f in files:
        p = os.path.join(CSRC, f)
        if os.path.isfile(p):
            h.update(f.encode())
            h.update(open(p, "rb").read())
    return h.hexdigest()


def build_library(force=False, verbose=False):
    os.makedirs(LIBDIR, exist_ok=True)
    stamp = os.path.join(LIBDIR, ".build_digest")
    dig = _digest()
    if not force and os.path.exists(LIB) and os.path.exists(stamp) and open(stamp).read() == dig:
        return LIB
    cmd = [_nvcc(), "-O3", "-std=c++17", "-lineinfo", *ARCH, "-shared", "-Xcompiler", "-fPIC,-O3",
           "-Xptxas", "-v" if verbose else "-O3",
           "-I", os.path.join(HERE, "..", "include"), "-o", LIB] + [os.path.join(CSRC, s) for s in SOURCES]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
        raise RuntimeError("nvcc failed building libdsmil_b200.so")
    if verbose:
        sys.stderr.write(r.stdout + r.stderr)
    with open(stamp, "w") as f:
        f.write(dig)
    return LIB


def _host_digest():
    h = hashlib.sha256()
    for f in sorted(os.listdir(HOST_CSRC)):
        h.update(f.encode())
        h.update(open(os.path.join(HOST_CSRC, f), "rb").read())
    h.update(open(os.path.join(CSRC, "jpeg_core.h"), "rb").read())      # shared with the device kernels
    return h.hexdigest()


def build_host_library(force=False):
    """libdsmil_host.so: host-only C (bag CSV reader / writer, csrc_host/), plain gcc -- no CUDA in it."""
    os.makedirs(LIBDIR, exist_ok=True)
    stamp = os.path.join(LIBDIR, ".build_digest_host")
    dig = _host_digest()
    if not force and os.path.exists(HOST_LIB) and os.path.exists(stamp) and open(stamp).read() == dig:
        return HOST_LIB
    cc = os.environ.get("CC") or shutil.which("gcc") or shutil.which("cc")
    if not cc:
        raise RuntimeError("no C compiler found (set CC=/path/to/gcc)")
    cmd = [cc, "-O3", "-std=c11", "-D_POSIX_C_SOURCE=200809L", "-Wall", "-Wextra", "-shared", "-fPIC", "-o", HOST_LIB] + \
          [os.path.join(HOST_CSRC, s) for s in HOST_SOURCES] + ["-lm", "-lpthread"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
        raise RuntimeError("gcc failed building libdsmil_host.so")
    with open(stamp, "w") as f:
        f.write(dig)
    return HOST_LIB


if __name__ == "__main__":
    print(build_library(force="--force" in sys.argv, verbose="-v" in sys.argv))
    print(build_host_library(force="--force" in sys.argv))
