"""`python -m ngp_pl_b200.train` end to end on the GPU, as a subprocess: the NeRF-synthetic lego fixture trained for two
epochs of 100 steps (files, the per-step scalar log, the checkpoints against an in-process evaluation and against the
reference's own utils.load_ckpt, --val_only), a short COLMAP run (the real-scene settings), and two ranks under torchrun
where the machine has two GPUs."""
import csv
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIX = os.path.join(ROOT, "tests", "golden", "datasets")


def _cli(args, cwd, prefix=None):
    env = {k: v for k, v in os.environ.items() if k not in ("WORLD_SIZE", "RANK", "LOCAL_RANK")}
    env["PYTHONPATH"] = ROOT + os.pathsep + env.get("PYTHONPATH", "")
    cmd = (prefix or [sys.executable, "-m"]) + ["ngp_pl_b200.train"] + args
    r = subprocess.run(cmd, cwd=cwd, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900)
    print(r.stdout[-3000:])
    assert r.returncode == 0, r.stdout[-3000:]
    return r.stdout


def _scalars(path):
    with open(path) as f:
        rows = list(csv.reader(f))
    head, steps, tests = rows[0], [], {}
    for r in rows[1:]:
        if r[0].startswith("test/"):
            tests[r[0]] = float(r[1])
        else:
            steps.append(dict(zip(head, [int(r[0])] + [float(v) for v in r[1:]])))
    return head, steps, tests


@pytest.fixture(scope="module")
def lego(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("cli_lego"))
    args = ["--root_dir", os.path.join(FIX, "lego"), "--dataset_name", "nerf", "--downsample", "0.1", "--num_epochs", "2",
            "--epoch_steps", "100", "--batch_size", "1024", "--exp_name", "lego", "--out_dir", out]
    log = _cli(args, cwd=out)
    return dict(out=out, args=args, log=log)


def test_lego_run_writes_the_reference_files_and_a_per_step_log(lego):
    from ngp_pl_b200.trainer import CosineAnnealingLR
    out = lego["out"]
    ck = os.path.join(out, "ckpts", "nerf", "lego")
    assert sorted(os.listdir(ck)) == ["epoch=1.ckpt", "epoch=1_slim.ckpt"]
    res = os.path.join(out, "results", "nerf", "lego")
    assert sorted(os.listdir(res)) == ["000.png", "000_d.png", "001.png", "001_d.png"]
    logs = os.path.join(out, "logs", "nerf", "lego")
    assert os.listdir(logs) == ["version_0"]
    head, steps, tests = _scalars(os.path.join(logs, "version_0", "scalars.csv"))
    assert head == ["step", "loss", "psnr", "rm_s", "vr_s", "lr"]
    assert [s["step"] for s in steps] == list(range(200))
    sch = CosineAnnealingLR(1e-2, T_max=2, steps_per_epoch=100)
    assert all(s["lr"] == float(np.float32(sch.lr_at_step(s["step"]))) for s in steps)
    assert all(s["rm_s"] > 0 and s["vr_s"] > 0 and np.isfinite(s["loss"]) for s in steps)
    first, last = np.mean([s["psnr"] for s in steps[:20]]), np.mean([s["psnr"] for s in steps[-20:]])
    assert last > first, (first, last)
    assert set(tests) == {"test/psnr", "test/ssim"} and tests["test/psnr"] > 10
    full = torch.load(os.path.join(ck, "epoch=1.ckpt"), weights_only=True)
    assert set(full) == {"epoch", "global_step", "state_dict"} and (full["epoch"], full["global_step"]) == (1, 200)
    sd = full["state_dict"]
    assert {"model.xyz_encoder.params", "model.rgb_net.params", "model.density_bitfield", "model.density_grid",
            "model.grid_coords", "directions", "poses"} <= set(sd)
    assert sd["directions"].shape == (80 * 80, 3) and sd["poses"].shape == (4, 3, 4)
    print(lego["log"].strip().splitlines()[-1])


def _model_from(path):
    from ngp_pl_b200 import train
    from ngp_pl_b200.models.networks import NGP
    model = NGP(0.5).cuda()
    G = model.grid_size
    model.register_buffer("density_grid", torch.zeros(model.cascades, G ** 3, device="cuda"))
    model.register_buffer("grid_coords", torch.zeros(G ** 3, 3, dtype=torch.int32, device="cuda"))
    train.load_weights(model, path)
    return model


def test_test_metrics_equal_an_evaluation_of_the_slim_checkpoint(lego, tmp_path):
    from ngp_pl_b200 import datasets, metrics
    out = lego["out"]
    model = _model_from(os.path.join(out, "ckpts", "nerf", "lego", "epoch=1_slim.ckpt"))
    test = datasets.load_scene("nerf", os.path.join(FIX, "lego"), "test", 0.1)
    res = metrics.evaluate(model, test.poses, test.directions, test.rgb, test.img_wh, save_dir=str(tmp_path))
    _, _, tests = _scalars(os.path.join(out, "logs", "nerf", "lego", "version_0", "scalars.csv"))
    assert res["psnr"] == tests["test/psnr"] and res["ssim"] == tests["test/ssim"], (res, tests)
    for f in ("000.png", "001_d.png"):
        with open(os.path.join(out, "results", "nerf", "lego", f), "rb") as a, open(str(tmp_path / f), "rb") as b:
            assert a.read() == b.read(), f


def test_val_only_reproduces_the_validation_pass(lego, tmp_path):
    out = lego["out"]
    args = ["--root_dir", os.path.join(FIX, "lego"), "--dataset_name", "nerf", "--downsample", "0.1", "--num_epochs", "2",
            "--epoch_steps", "100", "--exp_name", "lego_val", "--out_dir", str(tmp_path), "--val_only", "--ckpt_path",
            os.path.join(out, "ckpts", "nerf", "lego", "epoch=1.ckpt")]
    _cli(args, cwd=str(tmp_path))
    _, steps, tests = _scalars(os.path.join(str(tmp_path), "logs", "nerf", "lego_val", "version_0", "scalars.csv"))
    _, _, trained = _scalars(os.path.join(out, "logs", "nerf", "lego", "version_0", "scalars.csv"))
    assert steps == [] and tests["test/psnr"] == trained["test/psnr"]
    assert not os.path.exists(os.path.join(str(tmp_path), "ckpts"))
    a, b = os.path.join(out, "results", "nerf", "lego"), os.path.join(str(tmp_path), "results", "nerf", "lego_val")
    assert sorted(os.listdir(a)) == sorted(os.listdir(b))
    for f in os.listdir(a):
        with open(os.path.join(a, f), "rb") as x, open(os.path.join(b, f), "rb") as y:
            assert x.read() == y.read(), f


def test_reference_load_ckpt_reads_the_written_files(lego):
    """the reference's own utils.load_ckpt (staged byte-identical under oracle/_ref) loads both files into an NGP, and the
    model's state is the trained one"""
    import importlib.util
    path = os.path.join(ROOT, "oracle", "_ref", "ngp_pl", "utils.py")
    if not os.path.isfile(path):
        pytest.skip("the reference's utils.py is not staged under oracle/_ref")
    spec = importlib.util.spec_from_file_location("_ref_utils", path)
    utils = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(utils)
    from ngp_pl_b200.models.networks import NGP
    ck = os.path.join(lego["out"], "ckpts", "nerf", "lego")
    trained = torch.load(os.path.join(ck, "epoch=1.ckpt"), weights_only=True)["state_dict"]
    for name in ("epoch=1.ckpt", "epoch=1_slim.ckpt"):
        model = NGP(0.5).cuda()
        G = model.grid_size
        model.register_buffer("density_grid", torch.zeros(model.cascades, G ** 3, device="cuda"))
        model.register_buffer("grid_coords", torch.zeros(G ** 3, 3, dtype=torch.int32, device="cuda"))
        utils.load_ckpt(model, os.path.join(ck, name))
        sd = model.state_dict()
        skip = () if name == "epoch=1.ckpt" else ("density_grid", "grid_coords")
        for k, v in sd.items():
            if k not in skip:
                assert torch.equal(v.cpu(), trained["model." + k]), (name, k)


def test_colmap_run_uses_the_real_scene_settings(tmp_path):
    """--scale 16 on the 360_v2 fixture: exp_step_factor 1/256, black background, erode, and a finished run"""
    out = str(tmp_path)
    _cli(["--root_dir", os.path.join(FIX, "360_v2", "garden"), "--dataset_name", "colmap", "--scale", "16", "--num_epochs",
          "1", "--epoch_steps", "50", "--batch_size", "1024", "--exp_name", "garden", "--out_dir", out, "--no_save_test"],
         cwd=out)
    v = os.path.join(out, "logs", "colmap", "garden", "version_0")
    with open(os.path.join(v, "hparams.json")) as f:
        hp = json.load(f)["trainer"]
    assert hp["exp_step_factor"] == 1 / 256 and hp["bg"] == [0.0, 0.0, 0.0] and hp["erode"] and not hp["random_bg"]
    _, steps, tests = _scalars(os.path.join(v, "scalars.csv"))
    assert [s["step"] for s in steps] == list(range(50)) and np.isfinite(tests["test/psnr"])
    assert not os.path.exists(os.path.join(out, "results"))
    assert sorted(os.listdir(os.path.join(out, "ckpts", "colmap", "garden"))) == ["epoch=0.ckpt", "epoch=0_slim.ckpt"]


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_ranks_under_torchrun(tmp_path):
    out = str(tmp_path)
    _cli(["--root_dir", os.path.join(FIX, "lego"), "--dataset_name", "nerf", "--downsample", "0.1", "--num_epochs", "1",
          "--epoch_steps", "100", "--batch_size", "1024", "--exp_name", "lego2", "--out_dir", out, "--num_gpus", "2"],
         cwd=out, prefix=[sys.executable, "-m", "torch.distributed.run", "--standalone", "--nproc_per_node", "2", "-m"])
    _, steps, tests = _scalars(os.path.join(out, "logs", "nerf", "lego2", "version_0", "scalars.csv"))
    assert [s["step"] for s in steps] == list(range(100)) and tests["test/psnr"] > 10
    assert sorted(os.listdir(os.path.join(out, "results", "nerf", "lego2"))) == ["000.png", "000_d.png", "001.png", "001_d.png"]
