"""CPU-side checks of the drop-in boundary: libngp_b200.so loads, exports every symbol that
include/ngp_b200.h declares (no compute calls without a GPU), the ctypes binding read from the header agrees with
the C compiler and with bindings written out by hand, and the Python shim exposes the reference's twelve `vren` names."""
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "ngp_b200.h")


def declared_symbols():
    src = open(HEADER).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(ngp_[A-Za-z0-9_]+)\s*\(", src)))


def test_library_builds_and_exports_every_declared_symbol():
    from ngp_pl_b200 import build, _lib
    build.build()
    lib = _lib.lib()
    syms = declared_symbols()
    assert len(syms) >= 20
    for s in syms:
        assert hasattr(lib, s), "libngp_b200.so does not export " + s
    assert sorted(_lib.SIGNATURES.keys()) == syms, (
        "ctypes table and header disagree: %s" % (set(_lib.SIGNATURES.keys()) ^ set(syms)))
    assert lib.ngp_abi_version() == _lib.ABI_VERSION


def test_header_is_plain_c():
    import subprocess, tempfile
    with tempfile.TemporaryDirectory() as d:
        c = os.path.join(d, "t.c")
        open(c, "w").write('#include "ngp_b200.h"\nint main(void){return sizeof(NgpGridMeta)>0?0:1;}\n')
        r = subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.dirname(HEADER), "-c", c, "-o",
                            os.path.join(d, "t.o")], stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
        assert r.returncode == 0, r.stdout.decode()


def _probe(body):
    """stdout of a C program that includes the header and runs `body` in main"""
    import subprocess, tempfile
    with tempfile.TemporaryDirectory() as d:
        c = os.path.join(d, "t.c")
        open(c, "w").write('#include <stddef.h>\n#include <stdio.h>\n#include "ngp_b200.h"\n'
                           'int main(void){%s return 0;}\n' % body)
        exe = os.path.join(d, "t")
        subprocess.check_call(["gcc", "-I", os.path.dirname(HEADER), c, "-o", exe])
        return subprocess.check_output([exe]).decode().split()


def test_struct_layouts_match_header():
    """sizeof and the offsetof of every field of every struct, as the C compiler sees them == the ctypes mirrors"""
    import ctypes
    from ngp_pl_b200 import _lib
    names = re.findall(r"\}\s*(Ngp\w+)\s*;", open(HEADER).read())
    assert len(names) == 9
    want, body = [], ""
    for n in names:
        cls = getattr(_lib, n)
        want.append(("sizeof(%s)" % n, ctypes.sizeof(cls)))
        body += 'printf("%%zu\\n", sizeof(%s));' % n
        for f, _ in cls._fields_:
            want.append(("%s.%s" % (n, f), getattr(cls, f).offset))
            body += 'printf("%%zu\\n", offsetof(%s, %s));' % (n, f)
    got = [int(x) for x in _probe(body)]
    assert len(got) == len(want)
    for (what, py), c in zip(want, got):
        assert py == c, "%s: C says %d, ctypes says %d" % (what, c, py)


def test_defines_match_header():
    """every valued #define NGP_* is a constant of _lib with the value the C compiler gives it"""
    from ngp_pl_b200 import _lib
    names = re.findall(r"^#define[ \t]+(NGP_\w+)[ \t]+\S", open(HEADER).read(), re.M)
    assert len(names) >= 50
    got = _probe("".join('printf("%%.17g\\n", (double)(%s));' % n for n in names))
    for n, v in zip(names, got):
        assert getattr(_lib, n) == float(v), n
    assert _lib.ABI_VERSION == _lib.NGP_ABI_VERSION == 15
    assert _lib.NGP_INFER_FIELDS == ("t_cur", "t_end", "alive0", "alive1", "ray_start", "ray_n", "ray_idx", "ts", "deltas",
                                     "sigmas", "rgbs", "counters")


def test_bindings_read_from_header():
    """a few bindings written out by hand, one per kind of type the header reader maps"""
    import ctypes as C
    from ngp_pl_b200 import _lib
    S = _lib.SIGNATURES
    assert S["ngp_grid_meta"] == (C.c_uint32, [C.c_int, C.c_int, C.c_int, C.c_float, C.POINTER(_lib.NgpGridMeta)])
    assert S["ngp_launch_count"] == (C.c_ulonglong, [])
    assert S["ngp_splat_fit"][1][7] is C.c_double
    assert S["ngp_adam_step_fused"][1][5:7] == [C.c_uint64, C.c_uint64]
    assert S["ngp_render_infer_workspace"] == (C.c_size_t, [C.c_int, C.c_int64])
    assert S["ngp_render_train_fwd"][1][:3] == [C.POINTER(_lib.NgpNet), C.POINTER(_lib.NgpTrainCfg),
                                                C.POINTER(_lib.NgpTrainBuffers)]
    assert S["ngp_packbits"][1][0] is C.c_void_p and S["ngp_cast_params"][1][1] is C.c_void_p
    meta = dict(_lib.NgpGridMeta._fields_)
    assert meta["offset"]._type_ is C.c_uint32 and meta["offset"]._length_ == 17 and meta["scale"]._type_ is C.c_float
    assert _lib.NgpTrainCfg._fields_[:8] == [("n_rays", C.c_int32), ("cascades", C.c_int32), ("grid_size", C.c_int32),
                                             ("max_samples", C.c_int32), ("scale", C.c_float),
                                             ("exp_step_factor", C.c_float), ("T_threshold", C.c_float),
                                             ("near_distance", C.c_float)]
    assert [(f, t._length_) for f, t in _lib.NgpTrainCfg._fields_[8:11]] == [("center", 3), ("half_size", 3), ("bg", 3)]
    assert dict(_lib.NgpNet._fields_)["meta"] is _lib.NgpGridMeta
    assert dict(_lib.NgpNet._fields_)["enc_params_h"] is C.c_void_p


@pytest.mark.parametrize("decl, named", [
    ("int ngp_bad(long n, void* stream);", "ngp_bad"),
    ("typedef struct {\n    int32_t a;\n    long b;\n} NgpBad;", "NgpBad.b"),
    ("#define NGP_BAD (1 * 2)", "NGP_BAD"),
    ("#define NGP_BAD NGP_UNDEFINED", "NGP_BAD"),
    ("int ngp_bad(int a[4]);", "ngp_bad"),
])
def test_header_reader_refuses_what_it_cannot_map(tmp_path, decl, named):
    import ctypes as C
    from ngp_pl_b200 import _lib
    h = tmp_path / "bad.h"
    good = "#define NGP_ONE 1\n/* a comment */\nint ngp_ok(int n, void* stream);\n"
    h.write_text(good)
    assert _lib.parse_header(str(h)) == ({"NGP_ONE": 1}, {}, {"ngp_ok": (C.c_int, [C.c_int, C.c_void_p])})
    h.write_text(good + decl + "\n")
    with pytest.raises(RuntimeError, match=re.escape(named)) as e:
        _lib.parse_header(str(h))
    assert str(h) in str(e.value)


def test_header_reader_names_an_unreadable_header(tmp_path):
    from ngp_pl_b200 import _lib
    with pytest.raises(RuntimeError, match=re.escape(str(tmp_path / "missing.h"))):
        _lib.parse_header(str(tmp_path / "missing.h"))


def test_vren_surface():
    from ngp_pl_b200 import vren
    for name in ["ray_aabb_intersect", "ray_sphere_intersect", "packbits", "morton3D", "morton3D_invert",
                 "raymarching_train", "raymarching_test", "composite_train_fw", "composite_train_bw",
                 "composite_test_fw", "distortion_loss_fw", "distortion_loss_bw"]:
        assert callable(getattr(vren, name)), name


def test_grid_meta_tables_match_oracle(oracle):
    """level tables (host code, no GPU): product C-ABI vs the oracle restatement, BASELINE configs 1, 2, 5"""
    import numpy as np
    from ngp_pl_b200 import _lib
    for L, log2_T, scale in [(4, 14, 0.5), (16, 19, 0.5), (16, 19, 16.0), (16, 19, 2.0)]:
        b = float(np.exp(np.log(2048 * scale / 16) / (L - 1)))
        m, total = _lib.grid_meta(L, log2_T, 16, b)
        mo, total_o = oracle.grid_meta(L, log2_T, 16, float(np.float32(b)))
        assert total == total_o
        for l in range(L):
            assert m.res[l] == mo.res[l] and m.offset[l] == mo.offset[l] and m.scale[l] == mo.scale[l]
        assert m.hashed_mask == mo.hashed_mask
    m, total = _lib.grid_meta(16, 19, 16, float(np.exp(np.log(2048 * 0.5 / 16) / 15)))
    assert total == 5722520 and 2 * total + 3072 == 11448112  # SURVEY.md section 8, config C2
    assert list(m.res)[:6] == [16, 22, 28, 37, 49, 65] and m.res[15] == 1025


def test_ops_fail_loudly_without_gpu_or_library(monkeypatch):
    import torch
    from ngp_pl_b200 import vren, _lib
    if not torch.cuda.is_available():
        with pytest.raises(RuntimeError):
            vren.morton3D(torch.zeros(4, 3, dtype=torch.int32))  # CPU tensor: no CPU fallback
    monkeypatch.setattr(_lib, "_lib", None)
    monkeypatch.setattr(_lib, "LIB_PATH", "/nonexistent/libngp_b200.so")
    with pytest.raises(RuntimeError):
        _lib.lib()


def test_graft_entry_build_runs_on_cpu():
    """the driver's "does it build" check: __graft_entry__.build() compiles (cached) and imports everything without a GPU"""
    import importlib
    import os
    import sys
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    entry = importlib.import_module("__graft_entry__")
    entry.build()
