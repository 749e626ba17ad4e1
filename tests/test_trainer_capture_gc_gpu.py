"""Trainer.capture records its CUDA graphs with Python's automatic garbage collection off: torch.cuda.graph does not
collect before it begins, and a dead cycle holding an earlier Trainer's graphs, collected during a capture, would
destroy graphs where that is not permitted and invalidate the capture."""
import gc

import pytest
import torch

pytestmark = pytest.mark.gpu


def _trainer(seed):
    from ngp_pl_b200 import synth
    from ngp_pl_b200.models.networks import NGP
    from ngp_pl_b200.trainer import Trainer
    scene = synth.lego_scene(0)
    bank = synth.RayBank(scene, n_images=4, K=synth.intrinsics(W=100, H=100, fx=1111.11 / 8), device="cuda")
    torch.manual_seed(seed)
    tr = Trainer(NGP(scene.scale).cuda(), n_rays=4096, seed=seed)
    tr.attach_bank(bank)
    return tr


def test_capture_runs_without_automatic_collection_and_restores_it():
    old = _trainer(0)
    old.capture()
    old.train_step()
    old._cycle = old  # a deleted Trainer whose graphs only a collection frees
    del old
    tr = _trainer(1)
    seen = []
    prepare = tr._prepare

    def spy(*a, **k):
        seen.append((torch.cuda.is_current_stream_capturing(), gc.isenabled()))
        return prepare(*a, **k)

    tr._prepare = spy
    assert gc.isenabled()
    tr.capture()
    assert gc.isenabled()
    captured = [en for cap, en in seen if cap]
    assert captured and not any(captured)
    assert any(en for cap, en in seen if not cap)  # the eager warm-up step runs with collection on
    gc.collect()  # the old Trainer's graphs go now, outside any capture
    for _ in range(20):
        tr.train_step()
    torch.cuda.synchronize()
    assert torch.isfinite(torch.tensor(tr.stats()["loss"]))
