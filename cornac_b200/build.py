"""Build libb200cornac.so (sm_90a, H100) in-tree with nvcc.

    python -m cornac_b200.build [--force]

The shared library lands in cornac_b200/lib/ (git-ignored).  nvcc cross-compiles without a GPU.  No torch involved: the library is a plain
C-ABI .so (include/b200cornac.h) loaded with ctypes.
"""
import concurrent.futures
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "build")
LIBDIR = os.path.join(HERE, "lib")
LIB = os.path.join(LIBDIR, "libb200cornac.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
HOSTCXX = os.environ.get("B200_HOSTCXX", "/usr/bin/g++")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-std=c++17", "-lineinfo",
    "-ccbin", HOSTCXX,
    "-Xcompiler", "-fPIC,-fvisibility=hidden,-Wall",
    "--expt-relaxed-constexpr", "--expt-extended-lambda",
    "-Xptxas", "-v",
]


def sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith((".cu", ".cpp")))


def _stale(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def _compile(src, force):
    obj = os.path.join(OBJ, os.path.splitext(src)[0] + ".o")
    headers = [os.path.join(CSRC, h) for h in os.listdir(CSRC) if h.endswith((".cuh", ".h"))]
    headers.append(os.path.join(HERE, "..", "include", "b200cornac.h"))
    path = os.path.join(CSRC, src)
    if not force and not _stale(obj, [path] + headers):
        return obj, ""
    cmd = [NVCC] + NVCC_FLAGS + ["-c", path, "-o", obj]
    p = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if p.returncode != 0:
        raise RuntimeError("nvcc failed for %s:\n%s" % (src, p.stdout))
    with open(obj + ".log", "w") as f:
        f.write(p.stdout)
    return obj, p.stdout


def build(force=False, verbose=False):
    os.makedirs(OBJ, exist_ok=True)
    os.makedirs(LIBDIR, exist_ok=True)
    srcs = sources()
    with concurrent.futures.ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        results = list(ex.map(lambda s: _compile(s, force), srcs))
    objs = [r[0] for r in results]
    if verbose:
        for _, log in results:
            if log:
                print(log)
    if force or _stale(LIB, objs):
        cmd = [NVCC, "-shared", "-ccbin", HOSTCXX, "-gencode", "arch=compute_90a,code=sm_90a",
               "-o", LIB] + objs + ["-lcuda"]
        p = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        if p.returncode != 0:
            raise RuntimeError("link failed:\n" + p.stdout)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
