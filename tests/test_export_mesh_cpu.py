"""CPU tests of `python -m ngp_pl_b200.export_mesh`: its flags and defaults, and its refusals (exit status 2, naming
the flag, before torch is imported)."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _run(argv=None, code=None):
    cmd = [sys.executable, "-c", code] if code is not None else [sys.executable, "-m", "ngp_pl_b200.export_mesh"] + argv
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    return subprocess.run(cmd, cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=300)


def test_defaults_and_flags_parse_without_torch():
    code = ("import sys; from ngp_pl_b200 import export_mesh as E\n"
            "a = E.parse_args(['--ckpt_path', %r])\n"
            "print(a.scale, a.resolution, a.threshold, a.bounds, a.colors, a.no_normals, a.dense, a.out)\n"
            "b = E.parse_args(['--ckpt_path', %r, '--scale', '16', '--resolution', '8192', '--threshold', '0.5',"
            " '--bounds', '-1', '-2', '-3', '1', '2', '3', '--colors', '--no_normals', '--dense', '--out', 'x.ply'])\n"
            "print(b.scale, b.resolution, b.threshold, b.bounds, b.colors, b.no_normals, b.dense, b.out)\n"
            "print('torch' in sys.modules)\n" % (__file__, __file__))
    r = _run(None, code)
    assert r.returncode == 0, r.stderr
    lines = r.stdout.splitlines()
    assert lines[0] == "0.5 1024 20.0 None False False False mesh.ply"
    assert lines[1] == "16.0 8192 0.5 [-1.0, -2.0, -3.0, 1.0, 2.0, 3.0] True True True x.ply"
    assert lines[2] == "False"


def _refused(tmp):
    ok = os.path.join(tmp, "model_slim.ckpt")
    return [
        ([], "--ckpt_path"),
        (["--ckpt_path", os.path.join(tmp, "missing.ckpt")], "--ckpt_path"),
        (["--ckpt_path", os.path.join(tmp, "dir.ckpt")], "--ckpt_path"),
        (["--ckpt_path", ok, "--resolution", "1"], "--resolution"),
        (["--ckpt_path", ok, "--resolution", "8193"], "--resolution"),
        (["--ckpt_path", ok, "--threshold", "0"], "--threshold"),
        (["--ckpt_path", ok, "--threshold", "-5"], "--threshold"),
        (["--ckpt_path", ok, "--threshold", "nan"], "--threshold"),
        (["--ckpt_path", ok, "--bounds", "0", "0", "0", "1", "0", "1"], "--bounds"),
        (["--ckpt_path", ok, "--bounds", "0", "0", "0", "1", "-1", "1"], "--bounds"),
        (["--ckpt_path", ok, "--bounds", "0", "0", "0"], "--bounds"),
        (["--ckpt_path", ok, "--scale", "0"], "--scale"),
    ]


def test_refusals_exit_2_naming_the_flag(tmp_path):
    tmp = str(tmp_path)
    open(os.path.join(tmp, "model_slim.ckpt"), "wb").close()
    os.mkdir(os.path.join(tmp, "dir.ckpt"))
    for argv, flag in _refused(tmp):
        r = _run(argv)
        assert r.returncode == 2, (argv, r.returncode, r.stderr)
        assert flag in r.stderr, (argv, r.stderr)


def test_refusals_happen_before_torch(tmp_path):
    ok = os.path.join(str(tmp_path), "m.ckpt")
    open(ok, "wb").close()
    for argv in (["--ckpt_path", ok, "--threshold", "0"], ["--ckpt_path", ok, "--resolution", "9000"],
                 ["--ckpt_path", os.path.join(str(tmp_path), "missing.ckpt")]):
        code = ("import sys; from ngp_pl_b200 import export_mesh\n"
                "try:\n    export_mesh.main(%r)\n"
                "except SystemExit as e:\n    code = e.code\n"
                "print(code, 'torch' in sys.modules)\n" % (argv,))
        r = _run(None, code)
        assert r.stdout.split() == ["2", "False"], (argv, r.stdout, r.stderr)
