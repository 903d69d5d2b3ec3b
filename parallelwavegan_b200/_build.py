"""Build libpwgb.so in-tree with nvcc for sm_90a (no torch headers: pure C ABI)."""
import hashlib
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.path.join(HERE, "_lib")
LIB = os.path.join(LIBDIR, "libpwgb.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")


def _flags():
    return [
        "-gencode", "arch=compute_90a,code=sm_90a",
        "-O3", "-lineinfo", "-std=c++17",
        "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden",
        "-I", os.path.join(ROOT, "include"), "-I", CSRC,
    ]


def sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


def _digest():
    h = hashlib.sha256()
    for f in sources() + sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cuh")) + [
        os.path.join(ROOT, "include", "pwgb.h"), os.path.abspath(__file__)]:
        h.update(os.path.relpath(f, ROOT).encode())  # path-independent: the stamp built here stays valid on the GPU box
        with open(f, "rb") as fh:
            h.update(fh.read())
    return h.hexdigest()


def build(force=False, verbose=False):
    os.makedirs(LIBDIR, exist_ok=True)
    stamp = os.path.join(LIBDIR, "build.stamp")
    dig = _digest()
    if not force and os.path.exists(LIB) and os.path.exists(stamp) and open(stamp).read().strip() == dig:
        return LIB
    objs = []
    procs = []
    for src in sources():
        obj = os.path.join(LIBDIR, os.path.basename(src)[:-3] + ".o")
        cmd = [NVCC] + _flags() + (["-Xptxas", "-v"] if verbose else []) + ["-c", src, "-o", obj]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(obj)
    fail = False
    for src, pr in procs:
        out, _ = pr.communicate()
        if pr.returncode != 0:
            fail = True
            sys.stderr.write(f"[pwgb build] {src} failed:\n{out}\n")
        elif verbose or "warning" in out:
            sys.stderr.write(out)
    if fail:
        raise RuntimeError("nvcc failed building libpwgb.so")
    cmd = [NVCC, "-shared", "-o", LIB] + objs + ["-gencode", "arch=compute_90a,code=sm_90a", "-lcudart"]
    subprocess.check_call(cmd)
    with open(stamp, "w") as fh:
        fh.write(dig)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
