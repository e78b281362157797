"""In-tree build of libemu_b200.so (nvcc, sm_90a only).

The shared library is the product: a C-ABI (include/emu_b200.h) over hand-written CUDA.  It is built next to
the sources (emu_b200/libemu_b200.so) so that it travels to the GPU box with the repo snapshot.
"""
import hashlib
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libemu_b200.so")
STAMP = os.path.join(HERE, ".build_stamp")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC", "--use_fast_math=false" if False else "-DEMU_B200",
]


def sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


def _digest():
    h = hashlib.sha256()
    for f in sorted(os.listdir(CSRC)) + ["../../include/emu_b200.h"]:
        p = os.path.join(CSRC, f)
        if os.path.isfile(p):
            h.update(f.encode())
            h.update(open(p, "rb").read())
    return h.hexdigest()


def build(force=False, verbose=False):
    """Compile every .cu in csrc/ and link libemu_b200.so. Returns the library path."""
    dig = _digest()
    if not force and os.path.exists(LIB) and os.path.exists(STAMP) and open(STAMP).read() == dig:
        return LIB
    if not os.path.exists(NVCC):
        raise RuntimeError("nvcc not found at %s; cannot build libemu_b200.so" % NVCC)
    objdir = os.path.join(HERE, "build")
    os.makedirs(objdir, exist_ok=True)
    procs = []
    objs = []
    for src in sources():
        obj = os.path.join(objdir, os.path.basename(src)[:-3] + ".o")
        objs.append(obj)
        cmd = [NVCC] + FLAGS + ["-c", src, "-o", obj]
        if verbose:
            print(" ".join(cmd))
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)))
    failed = False
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            failed = True
            sys.stderr.write("nvcc failed for %s:\n%s\n" % (src, out.decode()))
        elif verbose and out:
            print(out.decode())
    if failed:
        raise RuntimeError("libemu_b200.so build failed")
    cmd = [NVCC, "-shared", "-o", LIB] + objs + ["-lcudart", "-ldl", "-gencode", "arch=compute_90a,code=sm_90a"]
    subprocess.check_call(cmd)
    with open(STAMP, "w") as f:
        f.write(dig)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
