"""Build the REAL reference (kwea123/ngp_pl) into oracle/_ref/  -- TEST INFRASTRUCTURE ONLY.

What this produces (all git-ignored, all under oracle/_ref/, nothing else is written):

  oracle/_ref/vren*.so        the reference's own CUDA extension `vren`, compiled from the sources
                              where they lie under /root/reference/models/csrc (binding.cpp,
                              raymarching.cu, volumerendering.cu, intersection.cu, losses.cu), for
                              sm_90 with the reference's own flags (-O2, models/csrc/setup.py:26-27).
  oracle/_ref/ngp_pl/         an *install* of the reference's Python hot-path modules
                              (models/{__init__,custom_functions,networks,rendering}.py, losses.py,
                              metrics.py), byte-identical, so `bench.py --impl reference` and the parity
                              tests can drive the UNMODIFIED reference `render()` on the GPU box, where
                              /root/reference does not exist.

The reference sources are never copied into the repository history: the scratch copy needed for the
13-site `.type()` -> `.scalar_type()` patch (torch>=2.x no longer converts DeprecatedTypeProperties
to ScalarType inside AT_DISPATCH_*; SURVEY.md section 8c) lives in a temporary directory.

The reference has NO CPU path (every op TORCH_CHECKs is_cuda, models/csrc/include/utils.h:4-6), so
this oracle only *runs* on the GPU box; it is *built* here (nvcc cross-compiles).

tinycudann is not vendored by the reference and is not installable here; the stand-in used when the
staged reference python does `import tinycudann` is oracle/tcnn_standin.py (parity UNPINNED for that
part, see DESIGN.md).
"""
import glob
import os
import re
import shutil
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get("NGP_REFERENCE_DIR", "/root/reference")
OUT = os.path.join(HERE, "_ref")

PY_FILES = [
    ("models/__init__.py", "ngp_pl/models/__init__.py"),
    ("models/custom_functions.py", "ngp_pl/models/custom_functions.py"),
    ("models/networks.py", "ngp_pl/models/networks.py"),
    ("models/rendering.py", "ngp_pl/models/rendering.py"),
    ("losses.py", "ngp_pl/losses.py"),
    ("metrics.py", "ngp_pl/metrics.py"),
]


def have_reference():
    return os.path.isdir(os.path.join(REF, "models", "csrc"))


def ref_vren_path():
    c = sorted(glob.glob(os.path.join(OUT, "vren*.so")))
    return c[0] if c else None


def stage_python():
    for src, dst in PY_FILES:
        d = os.path.join(OUT, dst)
        os.makedirs(os.path.dirname(d), exist_ok=True)
        shutil.copyfile(os.path.join(REF, src), d)


def build_vren(verbose=False):
    """nvcc/g++ directly on the reference's few source files (no reference build system)."""
    import torch
    from torch.utils import cpp_extension as ce

    csrc = os.path.join(REF, "models", "csrc")
    tmp = tempfile.mkdtemp(prefix="ngp_ref_build_")
    try:
        for f in os.listdir(csrc):
            p = os.path.join(csrc, f)
            if os.path.isfile(p) and (f.endswith(".cu") or f.endswith(".cpp")):
                s = open(p).read()
                if f.endswith(".cu"):
                    s = re.sub(r"\.type\(\)", ".scalar_type()", s)
                open(os.path.join(tmp, f), "w").write(s)
        inc = [os.path.join(csrc, "include")] + ce.include_paths("cuda")
        py_inc = subprocess.check_output(
            [sys.executable, "-c", "import sysconfig;print(sysconfig.get_paths()['include'])"]).decode().strip()
        inc.append(py_inc)
        iflags = sum((["-I", i] for i in inc), [])
        common = ["-DTORCH_EXTENSION_NAME=vren", "-DTORCH_API_INCLUDE_EXTENSION_H",
                  "-D_GLIBCXX_USE_CXX11_ABI=%d" % int(torch._C._GLIBCXX_USE_CXX11_ABI)]
        objs = []
        procs = []
        for f in sorted(os.listdir(tmp)):
            src = os.path.join(tmp, f)
            obj = src + ".o"
            if f.endswith(".cu"):
                cmd = ["nvcc", "-c", src, "-o", obj, "-O2", "-std=c++17",
                       "-gencode", "arch=compute_90,code=sm_90",
                       "--expt-relaxed-constexpr", "-Xcompiler", "-fPIC", "-w",
                       # the flags torch.utils.cpp_extension always adds for CUDAExtension
                       "-D__CUDA_NO_HALF_OPERATORS__", "-D__CUDA_NO_HALF_CONVERSIONS__",
                       "-D__CUDA_NO_BFLOAT16_CONVERSIONS__", "-D__CUDA_NO_HALF2_OPERATORS__"] + common + iflags
            elif f.endswith(".cpp"):
                cmd = ["g++", "-c", src, "-o", obj, "-O2", "-std=c++17", "-fPIC", "-w"] + common + iflags
            else:
                continue
            objs.append(obj)
            procs.append((f, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)))
        for f, p in procs:
            out, _ = p.communicate()
            if p.returncode != 0:
                raise RuntimeError("reference build failed on %s:\n%s" % (f, out.decode()[-4000:]))
            if verbose:
                print("[oracle/_ref] compiled", f)
        import sysconfig
        suffix = sysconfig.get_config_var("EXT_SUFFIX")
        os.makedirs(OUT, exist_ok=True)
        so = os.path.join(OUT, "vren" + suffix)
        libdirs = ce.library_paths("cuda")
        lflags = sum((["-L" + d, "-Wl,-rpath," + d] for d in libdirs), [])
        cmd = ["g++", "-shared", "-o", so] + objs + lflags + \
              ["-lc10", "-ltorch_cpu", "-ltorch", "-ltorch_python", "-lc10_cuda", "-ltorch_cuda", "-lcudart"]
        r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
        if r.returncode != 0:
            raise RuntimeError("reference link failed:\n" + r.stdout.decode()[-4000:])
        return so
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


def build(force=False, verbose=False):
    """Build oracle/_ref if the reference tree is present; otherwise use the prebuilt files."""
    if not have_reference():
        if ref_vren_path() is None:
            raise RuntimeError("no /root/reference and no prebuilt oracle/_ref/vren*.so")
        return ref_vren_path()
    stage_python()
    so = ref_vren_path()
    if so is not None and not force:
        newest = max(os.path.getmtime(p) for p in glob.glob(os.path.join(REF, "models", "csrc", "*.c*")))
        if os.path.getmtime(so) >= newest:
            return so
    return build_vren(verbose=verbose)


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
