"""Build librgcn_b200.so (sm_90a) in-tree with nvcc.

The shared library is the product's only compute path; it is built here (cross-compiled, no GPU
needed) and travels to the GPU box with the repository snapshot.
"""
import hashlib
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.path.join(HERE, "lib")
LIB = os.path.join(LIBDIR, "librgcn_b200.so")
SOURCES = ["graph.cu", "graph_device.cu", "rgcn_kernels.cu", "gemm_tf32x3.cu", "distmult.cu", "complex.cu", "basis_onehot.cu", "basis_diagcoef.cu", "gcn_diag.cu", "compgcn.cu", "highway.cu", "variational.cu", "topk.cu", "onen.cu", "self_adversarial.cu", "rotate.cu", "transe.cu", "quate.cu", "hole.cu", "conve.cu", "sampler.cu", "optimizer.cu", "block_staged.cu", "slice_norm.cu", "api.cu"]
HEADERS = ["graph.h", "kernels.cuh", "triple_rows.cuh", "dist_tile.cuh", os.path.join("..", "..", "include", "rgcn_b200.h")]


def _nvcc():
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found")


def _fingerprint():
    h = hashlib.sha256()
    for f in SOURCES + HEADERS:
        with open(os.path.join(CSRC, f), "rb") as fh:
            h.update(fh.read())
    return h.hexdigest()


def is_current():
    """True when the built library's stamp matches the sources' fingerprint."""
    stamp = os.path.join(LIBDIR, "librgcn_b200.stamp")
    if not (os.path.exists(LIB) and os.path.exists(stamp)):
        return False
    with open(stamp) as fh:
        return fh.read().strip() == _fingerprint()


def build(force=False, verbose=False):
    os.makedirs(LIBDIR, exist_ok=True)
    stamp = os.path.join(LIBDIR, "librgcn_b200.stamp")
    fp = _fingerprint()
    if not force and os.path.exists(LIB) and os.path.exists(stamp):
        with open(stamp) as fh:
            if fh.read().strip() == fp:
                return LIB
    cuda_home = os.path.dirname(os.path.dirname(_nvcc()))
    cmd = [
        _nvcc(), "-shared", "-Xcompiler", "-fPIC", "-O3", "-std=c++17", "-lineinfo", "--threads", "0",
        "-gencode", "arch=compute_90a,code=sm_90a",
        "-I", os.path.join(HERE, "..", "include"),
    ]
    if verbose:
        cmd += ["-Xptxas", "-v"]
    cmd += [os.path.join(CSRC, s) for s in SOURCES]
    cmd += ["-L", os.path.join(cuda_home, "lib64"), "-lcudart",
            "-Xlinker", "-rpath," + os.path.join(cuda_home, "lib64"), "-o", LIB]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        sys.stderr.write(res.stdout + res.stderr)
        raise RuntimeError("nvcc failed building librgcn_b200.so")
    if verbose:
        sys.stderr.write(res.stdout + res.stderr)
    with open(stamp, "w") as fh:
        fh.write(fp)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
