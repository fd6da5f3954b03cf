"""In-tree build of libedgedict_b200.so with nvcc for sm_90a (no torch headers, no pybind).

    python -m edgedict_b200.build            # incremental
    python -m edgedict_b200.build --force

The .so lands next to this file (git-ignored build product).
"""
import hashlib
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "build")
LIB = os.path.join(HERE, "libedgedict_b200.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
FLAGS = ARCH + ["-lineinfo", "-O3", "-std=c++17",
         "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden"]


def sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))


def _digest(path):
    h = hashlib.sha1()
    for dep in [path] + [os.path.join(CSRC, f) for f in sorted(os.listdir(CSRC)) if f.endswith(".cuh")] + \
            [os.path.join(HERE, "..", "include", f) for f in sorted(os.listdir(os.path.join(HERE, "..", "include")))]:
        with open(dep, "rb") as fh:
            h.update(fh.read())
    h.update(" ".join(FLAGS).encode())
    return h.hexdigest()


def _compile(src, force):
    path = os.path.join(CSRC, src)
    obj = os.path.join(OBJ, src[:-3] + ".o")
    stamp = obj + ".sha1"
    dg = _digest(path)
    if not force and os.path.exists(obj) and os.path.exists(stamp) and open(stamp).read() == dg:
        return obj, False
    cmd = [NVCC] + FLAGS + ["-c", path, "-o", obj]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("nvcc failed for %s:\n%s\n%s" % (src, r.stdout, r.stderr))
    with open(stamp, "w") as fh:
        fh.write(dg)
    return obj, True


def build(force=False, verbose=False):
    os.makedirs(OBJ, exist_ok=True)
    with ThreadPoolExecutor(max_workers=min(8, os.cpu_count() or 1)) as ex:
        res = list(ex.map(lambda s: _compile(s, force), sources()))
    objs = [o for o, _ in res]
    if force or any(c for _, c in res) or not os.path.exists(LIB):
        cmd = [NVCC, "-shared"] + ARCH + ["-o", LIB] + objs
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("link failed:\n%s\n%s" % (r.stdout, r.stderr))
        if verbose:
            print("linked", LIB)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
