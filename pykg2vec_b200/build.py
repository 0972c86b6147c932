"""Build libkge_b200.so in-tree with nvcc for sm_90a (H100; no JIT cache: the built
library is loaded from the source tree).

    python -m pykg2vec_b200.build [--force] [--verbose]
"""
import concurrent.futures
import glob
import hashlib
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT_DIR = os.path.join(HERE, "_build")
OBJ_DIR = os.path.join(OUT_DIR, "obj")  # intermediate objects (the SASS test reads them)
LIB = os.path.join(OUT_DIR, "libkge_b200.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr", "-Xptxas", "-v",
]


def _sources():
    return sorted(glob.glob(os.path.join(CSRC, "*.cu")))


def _stamp():
    h = hashlib.sha256()
    for p in sorted(glob.glob(os.path.join(CSRC, "*")) + [os.path.join(HERE, "..", "include", "kge_b200.h")]):
        with open(p, "rb") as f:
            h.update(os.path.basename(p).encode() + b"\0" + f.read())   # location-independent: a moved tree stays built
    h.update(" ".join(FLAGS).encode())
    return h.hexdigest()


def _compile(src, verbose):
    obj = os.path.join(OBJ_DIR, os.path.basename(src)[:-3] + ".o")
    cmd = [NVCC] + FLAGS + ["-c", src, "-o", obj]
    res = subprocess.run(cmd, capture_output=True, text=True)
    log = os.path.join(OUT_DIR, os.path.basename(src)[:-3] + ".ptxas.log")
    with open(log, "w") as f:
        f.write(res.stderr)
    if res.returncode != 0:
        raise RuntimeError("nvcc failed for %s:\n%s" % (src, res.stderr[-6000:]))
    if verbose:
        sys.stderr.write(res.stderr)
    return obj


def build(force=False, verbose=False):
    """Compile every .cu under csrc/ and link the C-ABI shared library. Returns its path."""
    os.makedirs(OBJ_DIR, exist_ok=True)
    stamp_file = os.path.join(OUT_DIR, "stamp.txt")
    stamp = _stamp()
    if not force and os.path.exists(LIB) and os.path.exists(stamp_file):
        with open(stamp_file) as f:
            if f.read().strip() == stamp:
                return LIB
    srcs = _sources()
    with concurrent.futures.ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        objs = list(ex.map(lambda s: _compile(s, verbose), srcs))
    cmd = [NVCC, "-shared", "-o", LIB + ".tmp"] + objs + ["-gencode", "arch=compute_90a,code=sm_90a",
                                                         "-cudart", "static"]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError("link failed:\n" + res.stderr[-4000:])
    os.replace(LIB + ".tmp", LIB)
    with open(stamp_file, "w") as f:
        f.write(stamp)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="--verbose" in sys.argv))
