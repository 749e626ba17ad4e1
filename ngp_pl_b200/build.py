"""In-tree build of libngp_b200.so (sm_90a only) with plain nvcc -- no torch headers, no JIT cache.

`python -m ngp_pl_b200.build` or `__graft_entry__.build()`. The .so and the object files are build products
(git-ignored).
"""
import hashlib
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
INCLUDE = os.path.join(os.path.dirname(HERE), "include")
HEADER = os.path.join(INCLUDE, "ngp_b200.h")
OBJ = os.path.join(HERE, "build")
LIB = os.path.join(HERE, "libngp_b200.so")

SOURCES = ["vren_ops.cu", "network.cu", "train.cu", "infer.cu", "modules.cu", "metrics.cu", "mesh.cu", "lpips.cu", "stage.cu", "images.cu", "jpeg.cu",
           "texture.cu", "points.cu", "components.cu", "fusion.cu", "splats.cu"]
# texture.cu's, points.cu's and fusion.cu's arithmetic must round operation by operation as their numpy restatements
# (oracle/mesh_texture.py, oracle/points_ref.py, oracle/tsdf_ref.py) do
SOURCE_FLAGS = {"texture.cu": ["-fmad=false"], "points.cu": ["-fmad=false"], "fusion.cu": ["-fmad=false"]}
NVCC_FLAGS = [
    "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo",
    "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr", "-Xptxas", "-v",
]


def _digest(paths):
    h = hashlib.sha256()
    for p in sorted(paths):
        h.update(p.encode())
        h.update(open(p, "rb").read())
    h.update(" ".join(NVCC_FLAGS).encode())
    h.update(repr(sorted(SOURCE_FLAGS.items())).encode())
    return h.hexdigest()


def sources():
    return [os.path.join(CSRC, s) for s in SOURCES if os.path.exists(os.path.join(CSRC, s))]


def build(force=False, verbose=False):
    srcs = sources()
    deps = srcs + [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cuh")] + [HEADER]
    stamp = os.path.join(OBJ, "stamp")
    dg = _digest(deps)
    if not force and os.path.exists(LIB) and os.path.exists(stamp) and open(stamp).read() == dg:
        return LIB
    os.makedirs(OBJ, exist_ok=True)

    def compile_one(src):
        obj = os.path.join(OBJ, os.path.basename(src) + ".o")
        cmd = ["nvcc", "-c", src, "-o", obj, "-I", INCLUDE] + NVCC_FLAGS + SOURCE_FLAGS.get(os.path.basename(src), [])
        r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
        log = r.stdout.decode()
        open(obj + ".log", "w").write(log)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed on %s:\n%s" % (src, log[-6000:]))
        if verbose:
            print(log)
        return obj

    with ThreadPoolExecutor(max_workers=4) as ex:
        objs = list(ex.map(compile_one, srcs))
    cmd = ["nvcc", "-shared", "-o", LIB] + objs + ["-gencode", "arch=compute_90a,code=sm_90a"]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
    if r.returncode != 0:
        raise RuntimeError("link failed:\n" + r.stdout.decode()[-4000:])
    open(stamp, "w").write(dg)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
