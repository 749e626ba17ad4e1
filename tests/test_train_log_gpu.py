"""The per-step training log (Trainer(log_rows=R), ngp_train_log_step, Trainer.drain_log) on the GPU: every drained row
equals the stats() of its step bitwise on each path of the step (eager and captured, fused loss, distortion loss,
same_image, random_bg, host batches through stage_batch, after_backward), the ring wraps and drains without losing or
reordering a row under the deep pipeline, an overrun raises, and with the log off the step is the step without it."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

N_RAYS = 4096


@pytest.fixture(scope="module")
def scene():
    from ngp_pl_b200 import synth
    s = synth.lego_scene(0)
    return s, synth.RayBank(s, n_images=8, device="cuda", seed=3)


def _trainer(scene, seed=0, **kw):
    from ngp_pl_b200.models.networks import NGP
    from ngp_pl_b200.trainer import Trainer
    s, bank = scene
    torch.manual_seed(seed)
    model = NGP(s.scale).cuda()
    tr = Trainer(model, n_rays=N_RAYS, seed=seed, **kw)
    tr.attach_bank(bank)
    return tr


PATHS = {
    "eager": dict(capture=False),
    "captured": dict(),
    "distortion": dict(trainer=dict(lambda_distortion=1e-3)),
    "same_image": dict(trainer=dict(ray_sampling_strategy="same_image")),
    "random_bg": dict(trainer=dict(random_bg=True)),
    "stage_batch": dict(sample=False),
    "after_backward": dict(after_backward=True),
    "eager_distortion": dict(capture=False, trainer=dict(lambda_distortion=1e-3)),
}


@pytest.mark.parametrize("path", sorted(PATHS))
def test_log_rows_equal_stats_bitwise(scene, path):
    from ngp_pl_b200.trainer import CosineAnnealingLR
    cfg = PATHS[path]
    sch = CosineAnnealingLR(1e-2, T_max=4, steps_per_epoch=10)
    tr = _trainer(scene, log_rows=16, lr_schedule=sch, **cfg.get("trainer", {}))
    sample = cfg.get("sample", True)
    bank = scene[1]
    batches = [bank.sample(N_RAYS) for _ in range(41)] if not sample else None
    hooked = []
    hook = (lambda t: hooked.append(t.host_step)) if cfg.get("after_backward") else None
    if not sample:
        tr.set_batch(*batches[0])
    if cfg.get("capture", True):
        tr.capture(sample=sample)
    if not sample:
        tr.stage_batch(*batches[0])
    stats, rows = [], []
    for k in range(40):
        tr.train_step(sample=sample, after_backward=hook)
        if not sample:
            tr.stage_batch(*batches[k + 1])
        torch.cuda.synchronize()
        stats.append(tr.stats())
        if k % 4 == 3:
            rows += tr.drain_log()
    rows += tr.drain_log(wait=True)
    assert [r["step"] for r in rows] == list(range(40))
    if hook is not None:
        assert len(hooked) == 40
    dist = tr.lambda_distortion > 0
    for k, (r, s) in enumerate(zip(rows, stats)):
        for key in ("rm_samples", "vr_samples", "bw_samples", "mse", "psnr") + (() if dist else ("loss",)):
            assert r[key] == s[key], (path, k, key, r[key], s[key])
        if dist:
            assert abs(r["distortion"] - s["distortion"]) <= 1e-6 * abs(s["distortion"]), (k, r["distortion"], s["distortion"])
            assert abs(r["loss"] - s["loss"]) <= 1e-6 * abs(s["loss"])
        assert r["lr"] == float(np.float32(sch.lr_at_step(k))), (k, r["lr"])
        assert np.isfinite(r["loss"])
    if sample:
        assert all(r["rm_samples"] > 0 for r in rows)
    assert len({r["lr"] for r in rows}) == 4


def test_ring_wraps_under_the_pipeline_without_losing_a_row(scene):
    """R = 8 over 40 captured steps, drained every 4 steps without any host synchronisation in between: every step once,
    in order, with the step index the device wrote"""
    tr = _trainer(scene, log_rows=8)
    tr.capture()
    rows = []
    for k in range(40):
        tr.train_step()
        if k % 4 == 3:
            rows += tr.drain_log()
    rows += tr.drain_log(wait=True)
    assert [r["step"] for r in rows] == list(range(40))
    assert all(r["rm_samples"] > 0 and r["vr_samples"] > 0 and np.isfinite(r["loss"]) for r in rows)
    # and with drains exactly R steps apart
    for k in range(16):
        tr.train_step()
        if k % 8 == 7:
            rows += tr.drain_log()
    rows += tr.drain_log(wait=True)
    assert [r["step"] for r in rows] == list(range(56))


def test_drain_after_more_than_R_steps_raises(scene):
    tr = _trainer(scene, log_rows=8)
    tr.capture()
    for _ in range(9):
        tr.train_step()
    with pytest.raises(RuntimeError, match="overwritten"):
        tr.drain_log()
    for _ in range(3):
        tr.train_step()
    assert [r["step"] for r in tr.drain_log(wait=True)] == [9, 10, 11]
    with pytest.raises(RuntimeError, match="off"):
        _trainer(scene).drain_log()


def _run(scene, steps, **kw):
    tr = _trainer(scene, seed=1, **kw)
    tr.capture()
    for _ in range(16):  # one refresh period: the launches per step are periodic in it
        tr.train_step()
    torch.cuda.synchronize()
    n0 = tr.launch_count()
    for _ in range(16):
        tr.train_step()
    per16 = tr.launch_count() - n0
    for _ in range(steps - 32):
        tr.train_step()
        if tr.log_ring is not None and tr.host_step % 8 == 0:
            tr.drain_log()
    torch.cuda.synchronize()
    return tr.P.clone(), per16


def test_log_off_changes_nothing(scene):
    """log_rows=0 is the trainer without the argument (same launches per step); with the log on the step launches one
    kernel more and trains to the same parameters -- bitwise, or, where two runs of the unchanged step differ (fp32
    atomics in the table gradient), within their spread"""
    a, na = _run(scene, 64)
    b, nb = _run(scene, 64, log_rows=0)
    c, nc = _run(scene, 64, log_rows=64)
    assert na == nb and nc == na + 16, (na, nb, nc)
    if torch.equal(a, b):
        assert torch.equal(c, a)
    else:
        spread = (a - b).abs().mean().item()
        assert (c - a).abs().mean().item() <= 3 * spread and (c - b).abs().mean().item() <= 3 * spread, spread
