"""The compositing kernels that share csrc/composite.cuh, held to exact equality.

- The Trainer's separate compositing kernels (k_train_composite_fw / k_train_composite_bw) and the vren operators
  (k_composite_train_fw / k_composite_train_bw) on the same samples. Both pairs index a ray's samples differently (int32
  offsets and counts against int64 rays_a) but composite them with the same arithmetic. With a zero background the
  Trainer's background terms add and subtract exact zeros, so the two paths do the same float operations and every
  output must be bitwise equal.
- The fused training kernel (k_train_composite_loss) with a non-zero background and a batch size whose reciprocal is
  not a power of two, against tests/golden/fused_composite.npz (tests/golden/make_golden_fused_composite.py): its
  per-ray outputs and per-sample gradients bit for bit, so a change to the order or rounding of its arithmetic -- such
  as how the background routes the colour gradient into the opacity gradient -- is seen, not only a change beyond the
  float64 bound of test_composite_fp64_gpu.py.
"""
import ctypes as C
import hashlib
import os

import numpy as np
import pytest
import torch

import cases
from test_fused_gpu import make_model

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("amp", [1.0, 16.0])
def test_trainer_separate_kernels_bitwise_equal_vren_operators(amp):
    """amp scales the random hash-table features: at 1 no ray of the batch reaches the transmittance threshold, at 16 about
    one in six does"""
    from ngp_pl_b200 import _lib, synth, vren
    from ngp_pl_b200.trainer import Trainer
    L_ = _lib.lib()
    scene = synth.lego_scene(0)
    n = 4096
    model = make_model(scene, amp=amp)
    o_np, d_np = cases.rays_from_scene(scene, n, 61, extra_edge_cases=True)
    o, d = torch.as_tensor(o_np).cuda(), torch.as_tensor(d_np).cuda()
    g = torch.Generator("cuda").manual_seed(5)
    gt = torch.rand(n, 3, device="cuda", generator=g)
    noise = torch.rand(n, device="cuda", generator=g)
    tr = Trainer(model, n_rays=n, bg=(0.0, 0.0, 0.0), fused_loss=False, materialize_ws=True)
    assert not tr.fused_loss and tr.ws is not None
    tr.set_batch(o, d, gt)
    tr.noise.copy_(noise)
    tr.march(jitter=False)
    tr.network()
    torch.cuda.synchronize()
    n_tot = int(tr.counters[0])
    assert n_tot > 0

    dC = torch.randn(n, 3, device="cuda", generator=g) * (0.5 / n)
    dOp = torch.randn(n, device="cuda", generator=g) * (1e-3 / n)
    dD = torch.randn(n, device="cuda", generator=g) * (0.3 / n)
    dws = torch.randn(tr.capacity, device="cuda", generator=g) * (1e-2 / n)
    ge = torch.zeros(tr.n_enc, device="cuda")
    gr = torch.zeros(tr.n_rgb, device="cuda")
    _lib.check(L_.ngp_render_train_bwd(C.byref(tr.net), C.byref(tr.cfg), C.byref(tr.buf), dC.data_ptr(),
                                       dOp.data_ptr(), dD.data_ptr(), dws.data_ptr(), ge.data_ptr(), gr.data_ptr(),
                                       tr._st()), "render_train_bwd")
    torch.cuda.synchronize()

    rays_a = torch.stack([torch.arange(n, device="cuda"), tr.offsets.long(), tr.n_samples.long()], 1).contiguous()
    sig, rgbs = tr.sigmas[:n_tot].contiguous(), tr.rgbs[:n_tot].contiguous()
    dl, ts = tr.deltas[:n_tot].contiguous(), tr.ts[:n_tot].contiguous()
    T = tr.cfg.T_threshold
    total, opacity, depth, rgb, ws = vren.composite_train_fw(sig, rgbs, dl, ts, rays_a, T)
    dsig, drgb = vren.composite_train_bw(dOp, dD, dC, dws[:n_tot].contiguous(), sig, rgbs, ws, dl, ts, rays_a,
                                         opacity, depth, rgb, T)
    torch.cuda.synchronize()

    def same(name, a, b):
        assert torch.equal(a, b), "%s: %d of %d differ" % (name, int((a != b).sum()), a.numel())

    assert int(tr.n_samples.sum()) == n_tot
    same("opacity", tr.opacity, opacity)
    same("depth", tr.depth, depth)
    same("rgb", tr.rgb.view(n, 3), rgb)
    same("ws", tr.ws[:n_tot], ws)
    same("dL/dsigma", tr.dsigmas[:n_tot], dsig)
    same("dL/drgb", tr.drgbs[:n_tot].reshape(n_tot, 3), drgb)
    # not vacuous: composited samples and non-zero gradients; with the denser field, rays that terminate (their
    # total_samples stops short of their sample count)
    terminated = int((total < tr.n_samples.long()).sum())
    print("amp %g: %d samples, %d composited, %d of %d rays terminated" % (amp, n_tot, int(total.sum()), terminated, n))
    assert int(total.sum()) > 0 and dsig.abs().max() > 0 and drgb.abs().max() > 0
    assert amp < 16 or terminated > n // 20


GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "fused_composite.npz")


def fused_step_outputs():
    """one ngp_render_train_step of a seeded 200-ray Lego batch with background (0.25, 0.5, 0.75) and lambda_opacity 1
    (so the opacity term and the routed colour gradient are of one size and the rounding of their difference shows);
    per-sample arrays in ray order (the marcher lays rays out in arrival order)"""
    from ngp_pl_b200 import synth
    from ngp_pl_b200.trainer import Trainer
    scene = synth.lego_scene(0)
    n = 200
    model = make_model(scene, amp=16.0)
    o_np, d_np = cases.rays_from_scene(scene, n, 67, extra_edge_cases=True)
    o, d = torch.as_tensor(o_np).cuda(), torch.as_tensor(d_np).cuda()
    g = torch.Generator("cuda").manual_seed(7)
    gt = torch.rand(n, 3, device="cuda", generator=g)
    noise = torch.rand(n, device="cuda", generator=g)
    tr = Trainer(model, n_rays=n, bg=(0.25, 0.5, 0.75), lambda_opacity=1.0)
    assert tr.fused_loss
    tr.set_batch(o, d, gt)
    tr.noise.copy_(noise)
    tr.march(jitter=False)
    tr._compute()
    torch.cuda.synchronize()
    cnt, off = tr.n_samples.long(), tr.offsets.long()
    idx = torch.repeat_interleave(off, cnt) + torch.arange(int(cnt.sum()), device="cuda") - \
        torch.repeat_interleave(torch.cumsum(cnt, 0) - cnt, cnt)
    net = torch.cat([tr.sigmas[idx], tr.rgbs[idx].reshape(-1)]).cpu().numpy()
    return dict(n_samples=cnt.int().cpu().numpy(), net_sha256=np.array(hashlib.sha256(net.tobytes()).hexdigest()),
                rgb=tr.rgb.cpu().numpy(), opacity=tr.opacity.cpu().numpy(), depth=tr.depth.cpu().numpy(),
                dsigmas=tr.dsigmas[idx].cpu().numpy(), drgbs=tr.drgbs[idx].cpu().numpy(),
                loss_scale=tr.scalars[1:2].cpu().numpy())


def test_fused_kernel_bitwise_equal_golden():
    ref = np.load(GOLDEN)
    got = fused_step_outputs()
    assert np.array_equal(got["n_samples"], ref["n_samples"]), "the marched batch changed"
    assert str(got["net_sha256"]) == str(ref["net_sha256"]), \
        "the network forward's outputs changed: regenerate with tests/golden/make_golden_fused_composite.py"
    for k in ("rgb", "opacity", "depth", "dsigmas", "drgbs", "loss_scale"):
        a, b = got[k], ref[k]
        assert a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32)), \
            "%s: %d of %d differ" % (k, int((a.view(np.uint32) != b.view(np.uint32)).sum()), b.size)
    # not vacuous: non-zero gradients, and rays that terminate
    assert np.abs(ref["dsigmas"]).max() > 0 and int((ref["opacity"] > 0.999).sum()) > 10
