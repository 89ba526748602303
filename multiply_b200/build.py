"""Build recipe of libmultiply_b200.so (explicit nvcc, sm_90a only, in-tree output).

    python -m multiply_b200.build [--force]

The .so and the objects under _build/ are build products (git-ignored); build() recompiles when a source changes.
"""
import os
import subprocess
import sys
import hashlib

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "libmultiply_b200.so")
OBJ = os.path.join(HERE, "_build")

ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
COMMON = ["-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC"]
# reference-semantics kernels: keep a*a + b*b as two roundings (see sampler.cu header).  mesh.cu too: its fp64
# closest-point and crossing arithmetic must round step by step as the CPU definitions' (oracle/mesh_port.py) do, so that
# distance types, tie-breaks and crossing parities agree exactly; mesh_extract.cu for the same reason (vertex
# positions, the asymptotic decider and component areas against oracle/mesh_extract.py); raster.cu for the same reason
# (projections, inside tests and depths against oracle/raster.py, distances against oracle/port.py:knn_points)
NO_FMAD = {"sampler.cu", "composite.cu", "rays.cu", "background.cu", "deform.cu", "mesh.cu", "mesh_extract.cu",
           "raster.cu"}
SOURCES = ["host_util.cu", "rays.cu", "deform.cu", "mlp_pack.cu", "mlp_simt.cu", "mlp_tc.cu", "mlp_grad.cu", "sampler.cu",
           "composite.cu", "background.cu", "render.cu", "smpl.cu", "mesh.cu", "mesh_extract.cu", "raster.cu"]


def _nvcc():
    for c in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if c and (os.path.isabs(c) and os.path.exists(c) or not os.path.isabs(c)):
            return c
    raise RuntimeError("nvcc not found")


def _stamp(path):
    h = hashlib.sha1()
    for f in sorted(os.listdir(CSRC)) + ["../../include/multiply_b200.h"]:
        with open(os.path.join(CSRC, f), "rb") as fh:
            h.update(fh.read())
    return h.hexdigest()


def build(force=False, verbose=False):
    os.makedirs(OBJ, exist_ok=True)
    stamp_file = os.path.join(OBJ, "stamp")
    stamp = _stamp(CSRC)
    if not force and os.path.exists(OUT) and os.path.exists(stamp_file) and open(stamp_file).read() == stamp:
        return OUT
    nvcc = _nvcc()
    objs = []
    procs = []
    for s in SOURCES:
        o = os.path.join(OBJ, s.replace(".cu", ".o"))
        cmd = [nvcc] + ARCH + COMMON + (["-fmad=false"] if s in NO_FMAD else []) + \
              ["-Xcompiler", "-DMP_BUILDING", "-c", os.path.join(CSRC, s), "-o", o]
        if verbose:
            print(" ".join(cmd))
        procs.append((s, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)))
        objs.append(o)
    for s, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            raise RuntimeError("nvcc failed on %s:\n%s" % (s, out.decode()))
        if verbose and out:
            print(out.decode())
    cmd = [nvcc] + ARCH + ["-shared", "-o", OUT] + objs + ["-lcudart", "-lcuda"]
    subprocess.check_call(cmd)
    with open(stamp_file, "w") as fh:
        fh.write(stamp)
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
