"""Build recipe for libdmnerf_b200.so (nvcc, sm_90a, built in-tree next to the package).

    python -m dmnerf_b200.build           # or __graft_entry__.build()
"""
import hashlib
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.path.join(HERE, "lib")
LIB = os.path.join(LIBDIR, "libdmnerf_b200.so")
SOURCES = ["abi.cu", "ray_kernels.cu", "mlp_simt.cu", "mlp_umma.cu", "backward.cu", "gemm_umma.cu", "penalizer.cu", "exchanger.cu", "evaluator.cu", "bwd_chain.cu", "mesh.cu", "metrics.cu", "inventory.cu", "components.cu", "region.cu", "collide.cu", "place.cu", "render_moves.cu", "raycast.cu", "edit_view.cu"]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
              "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden", "--expt-relaxed-constexpr"]


def nvcc():
    exe = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(exe):
        raise RuntimeError("nvcc not found (needed to build libdmnerf_b200.so)")
    return exe


def _digest():
    h = hashlib.sha256()
    files = sorted(os.listdir(CSRC)) + ["../../include/dmnerf_b200.h"]
    for f in files:
        with open(os.path.join(CSRC, f), "rb") as fh:
            h.update(f.encode()); h.update(fh.read())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def build(force=False, verbose=False):
    """Compile every .cu under csrc/ for sm_90a and link the shared library.  Returns the .so path."""
    os.makedirs(LIBDIR, exist_ok=True)
    stamp = os.path.join(LIBDIR, "build.sha256")
    dig = _digest()
    if not force and os.path.exists(LIB) and os.path.exists(stamp) and open(stamp).read().strip() == dig:
        return LIB
    objs = []
    procs = []
    for src in SOURCES:
        obj = os.path.join(LIBDIR, src.replace(".cu", ".o"))
        cmd = [nvcc()] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-c", os.path.join(CSRC, src), "-o", obj]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(obj)
    for src, p in procs:
        out, _ = p.communicate()
        if verbose or p.returncode:
            sys.stderr.write(out)
        if p.returncode:
            raise RuntimeError("nvcc failed on %s" % src)
    cmd = [nvcc(), "-shared", "-o", LIB] + objs + ["-lcudart"]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode:
        sys.stderr.write(r.stdout)
        raise RuntimeError("link failed")
    with open(stamp, "w") as f:
        f.write(dig)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
