"""The captured training step -- compute and optimiser in one CUDA graph, its kernels chained by programmatic dependent
launch (common.cuh) -- against the same step taken through the eager entry points with nothing overlapping: a one-thread
trace kernel after every kernel (ngp_trace_set) breaks each programmatic edge, and the host synchronises after every
call. Both start from identical state and the same marched batch, for several seeded batches.

What PDL may change: nothing but the order of the fp32 reductions. So the per-ray render, the loss scale, the live list
(as a set) and the per-sample feature gradients are bitwise equal; the hash-table gradient agrees within the rounding
bound of its two reduction orders; and the graph's optimiser, rerun synchronised on the gradient the graph itself
produced, gives bitwise the same parameters, moments and fp16 copy.

The optimiser runs with beta1 = 0.5 from zero moments, so that its first moment is exactly half the gradient it read: the
gradient inside the graph (consumed and cleared by the optimiser) is recovered bitwise from M.
"""
import numpy as np
import pytest
import torch

from oracle import grad64

pytestmark = pytest.mark.gpu

N_RAYS = 4096
N_BATCHES = 8


def _lib():
    from ngp_pl_b200 import _lib
    return _lib


@pytest.fixture(scope="module")
def setup():
    from ngp_pl_b200 import synth
    from ngp_pl_b200.models.networks import NGP
    from ngp_pl_b200.trainer import Trainer
    torch.manual_seed(0)
    scene = synth.lego_scene(0)
    model = NGP(scene.scale).cuda()
    with torch.no_grad():
        model.xyz_encoder.params[3072:].uniform_(-0.5, 0.5)  # O(1) features at every level
        model.density_bitfield.copy_(torch.as_tensor(synth.pack_bits(synth.occupancy_grid(scene))).cuda())
    bank = synth.RayBank(scene, n_images=8, device="cuda", seed=3)
    tr = Trainer(model, n_rays=N_RAYS, betas=(0.5, 0.75), update_interval=1 << 30)
    tr.host_step = 1  # no occupancy refresh
    tr.set_batch(*bank.sample(N_RAYS))
    tr.capture(sample=False)
    assert tr.g_step is not None
    torch.cuda.synchronize()
    return dict(tr=tr, bank=bank, model=model, P0=tr.P.clone(), Ph0=tr.Ph.clone())


def _reset(s, marched):
    tr = s["tr"]
    tr.P.copy_(s["P0"])
    tr.Ph.copy_(s["Ph0"])
    for t in (tr.M, tr.V, tr.G, tr.step_dev):
        t.zero_()
    tr.counters.copy_(marched["counters"])
    tr.scalars.copy_(marched["scalars"])
    torch.cuda.synchronize()


def _outputs(tr):
    n_live = int(tr.counters[5])
    live = tr.live_idx[:n_live].clone()
    order = torch.argsort(live)
    stride = (tr.capacity + 15) // 16 * 16
    L = int(tr.model.xyz_encoder.meta.n_levels)
    dfeat = tr.bwd_ws[:L * stride * 4].view(torch.int32).view(L, stride)[:, :n_live][:, order]
    return dict(rgb=tr.rgb.clone(), opacity=tr.opacity.clone(), depth=tr.depth.clone(), scale=tr.scalars[1].clone(),
                n_live=n_live, live=live[order], dfeat=dfeat.clone())


def _eager_step(tr):
    """the step's compute through its entry point, every kernel followed by a trace kernel (no programmatic overlap)"""
    _lib_ = _lib()
    buf = torch.zeros(2 + 2 * 64, dtype=torch.int64, device="cuda")
    buf[1] = 64
    _lib_.check(_lib_.lib().ngp_trace_set(buf.data_ptr()), "trace_set")
    try:
        tr._compute()
        torch.cuda.synchronize()
    finally:
        _lib_.lib().ngp_trace_set(None)
    assert int(buf[0]) >= 6  # stamps were enqueued between the kernels


def _eager_adam(tr, g):
    tr.G.copy_(g)
    torch.cuda.synchronize()
    _lib().check(_lib().lib().ngp_adam_step(tr.P.data_ptr(), tr.G.data_ptr(), tr.M.data_ptr(), tr.V.data_ptr(),
                                            tr.Ph.data_ptr(), tr.n_params, tr.lr_dev.data_ptr(), tr.step_dev.data_ptr(),
                                            tr.betas[0], tr.betas[1], tr.eps, 1.0, 1,
                                            torch.cuda.current_stream().cuda_stream), "adam")
    torch.cuda.synchronize()


@pytest.mark.parametrize("batch", range(N_BATCHES))
def test_graph_step_equals_serial_step(setup, batch):
    s = setup
    tr, bank = s["tr"], s["bank"]
    tr.set_batch(*bank.sample(N_RAYS))  # the next batch of the bank's seeded stream: a different one per parameter set
    tr.march(jitter=True)
    torch.cuda.synchronize()
    marched = dict(counters=tr.counters.clone(), scalars=tr.scalars.clone())

    _reset(s, marched)
    _eager_step(tr)
    ref = _outputs(tr)
    g_ref = tr.G.clone()
    assert ref["n_live"] > 0 and g_ref[3072:tr.n_enc].abs().max() > 0

    _reset(s, marched)
    tr._replay(tr.g_step[tr._cur][tr._gcur])
    torch.cuda.synchronize()
    got = _outputs(tr)
    after = {k: getattr(tr, k).clone() for k in ("P", "M", "V", "Ph")}
    assert int(tr.step_dev) == 1
    assert tr.G.abs().max() == 0, "the optimiser clears the gradient it consumed"

    for k in ("rgb", "opacity", "depth", "scale", "live", "dfeat"):
        assert torch.equal(got[k], ref[k]), k
    assert got["n_live"] == ref["n_live"]

    # the gradient the graph's optimiser read: M = (1 - beta1) * g = g / 2 exactly
    g_graph = after["M"] * 2
    n_enc = tr.n_enc
    # hash table: both sums lie within (m_e + 2) 2^-24 sum|contrib_e| of the exact one
    meta = tr.model.xyz_encoder.meta
    live = ref["live"].long()
    ridx = tr.ray_idx[live].long()
    x01 = (tr.rays_d[ridx].double() * tr.ts[live].double()[:, None] + tr.rays_o[ridx].double()).float() + 0.5
    dfeat16 = ref["dfeat"].t().contiguous().view(torch.float16).view(-1, 2 * int(meta.n_levels))
    _, Sabs, m = grad64.grid_scatter(meta, x01, dfeat16, 1.0 / float(ref["scale"]), tr.model.xyz_encoder.n_entries)
    tol = 2 * (m[:, None] + 2) * 2.0 ** -24 * Sabs
    diff = (g_graph[3072:n_enc].view(-1, 2).double() - g_ref[3072:n_enc].view(-1, 2).double()).abs()
    assert (diff <= tol).all(), "table gradient: %d entries outside the bound" % int((diff > tol).sum())
    # MLP weights: register accumulators flushed by fp32 reductions, one per CTA
    for a, b in ((g_graph[:3072], g_ref[:3072]), (g_graph[n_enc:], g_ref[n_enc:])):
        assert ((a - b).abs() <= 2.0 ** -14 * b.abs().max()).all()

    # the optimiser, rerun synchronised on the graph's own gradient
    _reset(s, marched)
    _eager_adam(tr, g_graph)
    for k in ("P", "M", "V", "Ph"):
        assert torch.equal(getattr(tr, k), after[k]), k


def test_back_to_back_graph_steps(setup):
    """200 sampled steps with no host synchronisation: finite loss, the step counter advances by exactly 200"""
    from ngp_pl_b200 import synth
    from ngp_pl_b200.models.networks import NGP
    from ngp_pl_b200.trainer import Trainer
    torch.manual_seed(0)
    scene = synth.lego_scene(0)
    model = NGP(scene.scale).cuda()
    tr = Trainer(model, n_rays=8192, update_interval=1 << 30)
    tr.host_step = 1
    tr.attach_bank(setup["bank"])
    tr.capture(sample=True)
    s0 = int(tr.step_dev)
    for _ in range(200):
        tr.train_step()
    torch.cuda.synchronize()
    assert int(tr.step_dev) - s0 == 200
    assert np.isfinite(tr.stats()["loss"])
    assert torch.isfinite(tr.P).all()
