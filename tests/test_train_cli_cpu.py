"""CPU tests of `python -m ngp_pl_b200.train` and of the host half of the per-step training log: the command line's flags
against the reference's own opt.py, the refused combinations (non-zero exit, a message naming the flag, no CUDA), the
Trainer settings a run derives from its flags, the checkpoint files against the reference's utils.py, and the ring's
index arithmetic and row decoding."""
import argparse
import importlib.util
import math
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "oracle", "_ref", "ngp_pl")


def _ref_module(name):
    path = os.path.join(REF, name + ".py")
    if not os.path.isfile(path):
        pytest.skip("the reference's %s.py is not staged under oracle/_ref" % name)
    spec = importlib.util.spec_from_file_location("_ref_" + name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _flags(parser):
    out = {}
    for a in parser._actions:
        if isinstance(a, argparse._HelpAction):
            continue
        out[a.dest] = dict(options=tuple(a.option_strings), kind=type(a).__name__, type=a.type, default=a.default,
                           choices=None if a.choices is None else list(a.choices), required=a.required)
    return out


def test_flags_match_the_reference_opt_py(monkeypatch):
    """every flag of the reference's opt.py, with its name, type, default and choices; the default dataset is the one
    deviation ('nsvf' is not loaded here)"""
    opt = _ref_module("opt")
    captured = {}

    def grab(self, *a, **k):
        captured["parser"] = self
        return argparse.Namespace()

    monkeypatch.setattr(argparse.ArgumentParser, "parse_args", grab)
    opt.get_opts()
    ref = _flags(captured["parser"])
    monkeypatch.undo()
    from ngp_pl_b200 import train
    ours = _flags(train.get_parser())
    assert len(ref) >= 20
    for dest, spec in ref.items():
        assert dest in ours, "flag --%s of the reference is missing" % dest
        got = dict(ours[dest])
        if dest == "dataset_name":
            assert spec["default"] == "nsvf" and got["default"] == "nerf"
            got["default"] = spec["default"]
        assert got == spec, (dest, got, spec)
    assert set(ours) - set(ref) == {"seed", "out_dir", "epoch_steps", "lpips_vgg", "lpips_lin", "video_fps"}


REFUSED = [
    (["--dataset_name", "nsvf"], "--dataset_name"),
    (["--dataset_name", "nerfpp"], "--dataset_name"),
    (["--dataset_name", "rtmv"], "--dataset_name"),
    (["--use_exposure"], "--use_exposure"),
    (["--optimize_ext"], "--optimize_ext"),
    (["--split", "trainvaltest"], "--split"),
    (["--eval_lpips"], "--lpips_vgg"),
    (["--eval_lpips", "--lpips_vgg", __file__], "--lpips_lin"),
    (["--num_gpus", "2"], "--num_gpus"),
    (["--ckpt_path", "x.ckpt"], "--ckpt_path"),
    (["--val_only"], "--val_only"),
]


@pytest.mark.parametrize("argv,flag", REFUSED, ids=[" ".join(a) for a, _ in REFUSED])
def test_refused_combinations_exit_nonzero_naming_the_flag(argv, flag):
    env = {k: v for k, v in os.environ.items() if k not in ("WORLD_SIZE", "RANK", "LOCAL_RANK")}
    env["PYTHONPATH"] = ROOT + os.pathsep + env.get("PYTHONPATH", "")
    r = subprocess.run([sys.executable, "-m", "ngp_pl_b200.train", "--root_dir", "does/not/exist"] + argv, cwd=ROOT, env=env,
                       stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=120)
    assert r.returncode != 0
    assert flag in r.stderr, r.stderr


def test_refusals_happen_before_torch_or_cuda():
    """the checks run on the parsed flags alone: torch is not even imported"""
    code = ("import sys; from ngp_pl_b200 import train\n"
            "try:\n    train.main(['--root_dir', 'x', '--use_exposure'])\nexcept SystemExit as e:\n    code = e.code\n"
            "print(code, 'torch' in sys.modules)\n")
    env = {k: v for k, v in os.environ.items() if k != "WORLD_SIZE"}
    env["PYTHONPATH"] = ROOT + os.pathsep + env.get("PYTHONPATH", "")
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.PIPE,
                       text=True, timeout=120)
    assert r.stdout.split() == ["2", "False"], (r.stdout, r.stderr)


def test_num_gpus_must_match_the_torchrun_world():
    from ngp_pl_b200 import train
    p = train.get_parser()
    args = p.parse_args(["--root_dir", "x", "--num_gpus", "2"])
    assert train.check_args(args, p, environ={"WORLD_SIZE": "2"}) is args
    with pytest.raises(SystemExit):
        train.check_args(p.parse_args(["--root_dir", "x", "--num_gpus", "2"]), p, environ={"WORLD_SIZE": "4"})
    with pytest.raises(SystemExit):
        train.check_args(p.parse_args(["--root_dir", "x"]), p, environ={"WORLD_SIZE": "2"})


def test_trainer_settings_follow_the_reference_train_py():
    from ngp_pl_b200 import train
    p = train.get_parser()
    s = train.trainer_settings(p.parse_args(["--root_dir", "x"]))
    assert s["exp_step_factor"] == 0 and s["bg"] == (1.0, 1.0, 1.0) and not s["random_bg"] and not s["erode"]
    assert s["n_rays"] == 8192 and s["lr"] == 1e-2 and s["lambda_distortion"] == 0
    sch = s["lr_schedule"]
    assert (sch.T_max, sch.steps_per_epoch, sch.base_lr, sch.eta_min) == (30, 1000, 1e-2, 1e-2 / 30)
    # synthetic scenes keep the white background even with --random_bg (rendering.py:153-161)
    assert not train.trainer_settings(p.parse_args(["--root_dir", "x", "--random_bg"]))["random_bg"]
    s = train.trainer_settings(p.parse_args(["--root_dir", "x", "--dataset_name", "colmap", "--scale", "16",
                                             "--random_bg", "--distortion_loss_w", "1e-3", "--batch_size", "4096",
                                             "--ray_sampling_strategy", "same_image", "--num_epochs", "5",
                                             "--epoch_steps", "100", "--lr", "2e-2"]))
    assert s["exp_step_factor"] == 1 / 256 and s["bg"] == (0.0, 0.0, 0.0) and s["random_bg"] and s["erode"]
    assert s["lambda_distortion"] == 1e-3 and s["n_rays"] == 4096 and s["ray_sampling_strategy"] == "same_image"
    sch = s["lr_schedule"]
    assert (sch.T_max, sch.steps_per_epoch, sch.base_lr) == (5, 100, 2e-2)
    assert sch.lr_at_step(99) == 2e-2 and sch.lr_at_step(100) < 2e-2


# ---- checkpoints ----------------------------------------------------------------------------------------------------------
def _toy_model():
    import torch
    m = torch.nn.Module()
    m.lin = torch.nn.Linear(3, 2)
    m.register_buffer("density_grid", torch.rand(2, 8))
    m.register_buffer("grid_coords", torch.arange(24, dtype=torch.int32).reshape(8, 3))
    m.register_buffer("density_bitfield", torch.randint(0, 255, (4,), dtype=torch.uint8))
    return m


def test_checkpoint_files_against_the_reference_utils(tmp_path):
    """the slim file is the reference's slim_ckpt of the full one, and the reference's load_ckpt and ours load either
    into a model identically"""
    import torch
    utils = _ref_module("utils")
    from ngp_pl_b200 import train
    torch.manual_seed(0)
    m = _toy_model()
    ck = train.checkpoint(m, torch.rand(6, 3), torch.rand(2, 3, 4), 1, 200)
    assert set(ck) == {"epoch", "global_step", "state_dict"} and (ck["epoch"], ck["global_step"]) == (1, 200)
    assert set(ck["state_dict"]) == {"model." + k for k in m.state_dict()} | {"directions", "poses"}
    full, slim = str(tmp_path / "epoch=1.ckpt"), str(tmp_path / "epoch=1_slim.ckpt")
    torch.save(ck, full)
    torch.save(train.slim_state_dict(ck), slim)
    ref_slim = utils.slim_ckpt(full)
    ours = torch.load(slim, weights_only=True)
    assert list(ours) == list(ref_slim) and all(torch.equal(ours[k], ref_slim[k]) for k in ours)
    for path in (full, slim):
        torch.manual_seed(1)
        a = _toy_model()
        torch.manual_seed(1)
        b = _toy_model()
        utils.load_ckpt(a, path)
        train.load_weights(b, path)
        sa, sb = a.state_dict(), b.state_dict()
        assert all(torch.equal(sa[k], sb[k]) for k in sa)
        assert torch.equal(sa["lin.weight"], m.lin.weight.detach())


# ---- the log ring ---------------------------------------------------------------------------------------------------------
def test_ring_spans_cover_the_steps_in_order():
    from ngp_pl_b200.trainer import log_ring_spans
    for R in (1, 3, 8, 256):
        for first in range(0, 3 * R + 2):
            for n in range(0, R + 1):
                spans = log_ring_spans(first, n, R)
                rows = [r for lo, hi in spans for r in range(lo, hi)]
                assert rows == [(first + k) % R for k in range(n)]
                assert len(spans) <= 2 and all(0 <= lo < hi <= R for lo, hi in spans)
    with pytest.raises(RuntimeError):
        log_ring_spans(5, 9, 8)


def test_simulated_ring_drains_lose_and_reorder_nothing():
    """the device writes step k at row k % R; draining every d steps with the host's spans returns every step once, in
    order, while d <= R, and the first drain after more than R steps would need rows already overwritten"""
    from ngp_pl_b200.trainer import log_ring_spans
    rng = np.random.RandomState(0)
    for R in (1, 4, 8, 13):
        ring = np.full(R, -1)
        got, nxt = [], 0
        for step in range(5 * R + 7):
            ring[step % R] = step
            if rng.rand() < 0.4 or step - nxt + 1 == R:
                n = step + 1 - nxt
                got += [int(v) for lo, hi in log_ring_spans(nxt, n, R) for v in ring[lo:hi]]
                nxt = step + 1
        assert got == list(range(nxt))
        with pytest.raises(RuntimeError):
            log_ring_spans(0, R + 1, R)


def test_log_rows_decode_with_the_formulas_of_stats():
    """loss, mse and psnr are computed from the rows' fp32 values exactly as Trainer.stats() computes them from the
    device tensors' values"""
    from ngp_pl_b200.trainer import log_rows_to_stats
    rng = np.random.RandomState(1)
    n, lam = 4096, float(np.float32(1e-3))
    rows = np.zeros((5, 8), np.int32)
    f = rows.view(np.float32)
    f[:, 0] = rng.rand(5).astype(np.float32) * 100
    f[:, 1] = rng.rand(5).astype(np.float32) * 50
    rows[:, 2:5] = rng.randint(0, 10 ** 6, (5, 3))
    f[:, 5] = np.float32(0.01)
    f[:, 6] = rng.rand(5).astype(np.float32)
    rows[:, 7] = np.arange(10, 15)
    rows[0, 0] = 0  # sse 0: psnr of the 1e-12 floor
    for live in (True, False):
        for dist in (0.0, 1e-2):
            out = log_rows_to_stats(rows, n, lam, dist, live)
            for r, x, d in zip(rows.tolist(), f.tolist(), out):
                mse = x[0] / (3 * n)
                loss = mse + lam * x[1] / n
                assert d["mse"] == mse and d["psnr"] == -10 * math.log10(max(mse, 1e-12))
                assert (d["rm_samples"], d["vr_samples"], d["bw_samples"]) == (r[2], r[3], r[4] if live else r[2])
                assert d["step"] == r[7] and d["lr"] == float(np.float32(0.01))
                if dist:
                    assert d["distortion"] == dist * (x[6] / n) and d["loss"] == loss + d["distortion"]
                else:
                    assert "distortion" not in d and d["loss"] == loss
