"""The optimiser kernels, element by element, against the float64 Adam restatement oracle/adam64.py.

Every call is checked from the kernel's own inputs: m' and v' within 2 x their bounds, p' within 2 x its bound computed
from the kernel's own m' and v', the fp16 working copy bitwise __float2half_rn(p'), the gradient exactly zero afterwards
where the kernel owns the clear, and the step counter advanced by increment_step.

  * ngp_adam_step (k_adam) at sizes taken from the SM count, so that every path of its loop runs -- one group per
    thread, a second group for some threads only, several trips with a partial last one, each with a scalar tail of
    0-3 -- and at the Trainer's 11,455,280 parameters; over step counters 1 .. 10^5, three beta pairs, two eps, three
    gradient multipliers and learning rates changed on the device between calls, with gradients from 1e-25 to 1e4;
  * the skip of untouched float4 groups (g = m = v = 0: nothing is stored) against groups that must still be updated;
  * params_half = NULL, argument rejection, n = 0;
  * the exchange kernels ngp_adam_step_fused and ngp_adam_step_p2p with world = 1 (the peer arrays are the local
    buffers, the barriers meet themselves): within the bound and bitwise equal to ngp_adam_step, the next gradient
    buffer cleared, the consumed one untouched, the epochs advanced by one per call -- eagerly and over CUDA-graph
    replays;
  * the Trainer's wiring: after a captured step on the Lego scene, P, M and V within the bound of the float64 step from
    a snapshot of G, P, M, V, lr and the counter taken between the backward and the optimiser.
"""
import ctypes as C

import pytest
import torch

from oracle import adam64 as A

pytestmark = pytest.mark.gpu

EINVAL = -22
RATIOS = {}     # output -> largest error / (SAFETY bound) over the module's calls
WORST_P = {}    # (beta2, t) -> largest p' ratio


def note(name, r):
    RATIOS[name] = max(RATIOS.get(name, 0.0), r)
    assert r <= 1.0, "%s: error / (%g x bound) = %.3g" % (name, A.SAFETY, r)


@pytest.fixture(scope="module", autouse=True)
def report():
    yield
    print("\nAdam vs float64, largest error / (%g x bound):" % A.SAFETY)
    for k in sorted(RATIOS):
        print("  %-24s %.3g" % (k, RATIOS[k]))
    if WORST_P:
        print("  p' by (beta2, t):", ", ".join("(%g, %d) %.3g" % (b, t, r) for (b, t), r in sorted(WORST_P.items())))


def _L():
    from ngp_pl_b200 import _lib
    return _lib.lib()


def _st():
    return torch.cuda.current_stream().cuda_stream


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.fixture(scope="module")
def pool():
    """one seeded state of 11,455,283 elements on the device, sliced by the tests"""
    return tuple(x.cuda() for x in A.random_state(11455280 + 3, seed=5))


class State:
    """fp32 parameters, gradient, moments and an fp16 copy prefilled with a sentinel (NaN), plus lr and the counter"""

    def __init__(self, p, g, m, v, t=1, lr=1e-2, ph=None):
        self.P, self.G, self.M, self.V = (x.clone().contiguous() for x in (p, g, m, v))
        self.Ph = torch.full_like(self.P, float("nan"), dtype=torch.float16) if ph is None else ph.clone()
        self.lr = torch.tensor([lr], dtype=torch.float32, device="cuda")
        self.step = torch.tensor([t - 1], dtype=torch.int32, device="cuda")

    def clone(self):
        s = State(self.P, self.G, self.M, self.V, ph=self.Ph)
        s.lr, s.step = self.lr.clone(), self.step.clone()
        return s

    def tensors(self):
        return dict(P=self.P, G=self.G, M=self.M, V=self.V, Ph=self.Ph, step=self.step)


def adam_step(s, n, b1, b2, eps, gm, inc=1, ph=True):
    return _L().ngp_adam_step(s.P.data_ptr(), s.G.data_ptr(), s.M.data_ptr(), s.V.data_ptr(),
                              s.Ph.data_ptr() if ph else None, n, s.lr.data_ptr(), s.step.data_ptr(), b1, b2, eps, gm,
                              inc, _st())


def check_call(label, before, after, n, b1, b2, eps, gm, ph="all", grad_cleared=True, inc=1):
    """after = the kernel's result from `before` (State snapshots). ph: 'all' -- every element's fp16 copy is half(p');
    'skip' -- groups with g = m = v = 0 keep their old fp16 value and p, m, v bitwise; None -- not written."""
    t = int(before.step) + 1
    lr = float(before.lr)
    P0, G0, M0, V0 = (x[:n] for x in (before.P, before.G, before.M, before.V))
    P1, M1, V1 = (x[:n] for x in (after.P, after.M, after.V))
    o = A.step(P0, G0, M0, V0, t, lr, b1, b2, eps, gm, m_k=M1, v_k=V1)
    rm = A.ratio(M1.double() - o["m"], o["m_err"])
    rv = A.ratio(V1.double() - o["v"], o["v_err"])
    rp = A.ratio(P1.double() - o["p"], o["p_err"])
    key = (A.f32(b2), t)
    WORST_P[key] = max(WORST_P.get(key, 0.0), rp)
    for name, r in (("m'", rm), ("v'", rv), ("p'", rp)):
        note(name, r)
    assert int(after.step) == int(before.step) + inc, label
    if grad_cleared and n:
        assert after.G[:n].abs().max().item() == 0, label + ": the gradient must be cleared"
    if ph is None:
        return
    want = P1.half().view(torch.int16)
    got = after.Ph[:n].view(torch.int16)
    if ph == "skip":
        n4 = n // 4
        untouched = torch.zeros(n, dtype=torch.bool, device="cuda")
        zero = ((G0[:4 * n4] == 0) & (M0[:4 * n4] == 0) & (V0[:4 * n4] == 0)).view(n4, 4).all(1)
        untouched[:4 * n4] = zero.repeat_interleave(4)
        want = torch.where(untouched, before.Ph[:n].view(torch.int16), want)
        for x0, x1 in ((P0, P1), (M0, M1), (V0, V1)):
            assert torch.equal(x0[untouched].view(torch.int32), x1[untouched].view(torch.int32)), label
    assert torch.equal(got, want), label + ": fp16 copy differs from half(p') at %d elements" % int((got != want).sum())


def run_adam(label, s, n, b1=0.9, b2=0.999, eps=1e-15, gm=1.0):
    before = s.clone()
    assert adam_step(s, n, b1, b2, eps, gm) == 0
    torch.cuda.synchronize()
    check_call(label, before, s, n, b1, b2, eps, gm, ph="skip")


def loop_sizes():
    """(n4, tail) covering k_adam's loop: the grid is min(ceil((n4 + 1) / 256), 2 SMs) blocks of 256 threads, each thread
    takes groups i0 and i0 + stride per trip and advances by two strides"""
    T = 2 * sms() * 256
    n4s = [T // 2 + 3, T - 1,             # below one stride: one group per thread
           T + 5, T + T // 2, 2 * T - 1,  # between one and two strides: `two` false for some threads
           2 * T, 2 * T + 1,              # one full trip, then a partial one
           3 * 2 * T + T // 3,            # several trips, the last one without a second group
           3 * 2 * T + T + T // 2]        # several trips, the last one's second group for some threads
    return [(n4, tail) for n4 in n4s for tail in range(4)]


@pytest.mark.parametrize("n", [1, 2, 3, 4, 5, 7, 8])
def test_adam_tiny_sizes(pool, n):
    p, g, m, v = pool
    run_adam("n=%d" % n, State(p[:n], g[:n], m[:n], v[:n], t=2), n)


def test_adam_loop_sizes(pool):
    p, g, m, v = pool
    for k, (n4, tail) in enumerate(loop_sizes()):
        n = 4 * n4 + tail
        o = (977 * k) % 1000  # a different slice of the pool per size
        s = State(p[o:o + n], g[o:o + n], m[o:o + n], v[o:o + n], t=1 + k % 3)
        run_adam("n4=%d tail=%d" % (n4, tail), s, n, gm=0.5 if k % 2 else 1.0 / 3)


def test_adam_trainer_size(pool):
    p, g, m, v = pool
    n = 11455280
    run_adam("n=%d" % n, State(p[:n], g[:n], m[:n], v[:n], t=3), n, eps=1e-15, gm=1.0)


def test_adam_state_grid(pool):
    """counters 1 .. 10^5, three beta pairs, eps 1e-15 / 1e-8, grad_mul 1, 1/2, 1/3; lr rewritten on the device before
    every call; the same state buffers carried from call to call"""
    p, g, m, v = pool
    n = 4 * 4099 + 3
    k = 0
    for t in (1, 2, 3, 5, 10, 100, 10 ** 4, 10 ** 5):
        for b1, b2 in ((0.9, 0.999), (0.9, 0.99), (0.5, 0.75)):
            for eps in (1e-15, 1e-8):
                for gm in (1.0, 0.5, 1.0 / 3):
                    o = 4099 * k
                    s = State(p[o:o + n], g[o:o + n], m[o:o + n], v[o:o + n], t=t)
                    s.lr.fill_(1e-2 * (1 + k % 7) / 4)
                    run_adam("t=%d betas=(%g, %g) eps=%g grad_mul=%g" % (t, b1, b2, eps, gm), s, n, b1, b2, eps, gm)
                    k += 1


def test_adam_moments_carried_over_steps(pool):
    """five consecutive calls on one state (the counter advanced by the kernel's own increment), lr changed in between"""
    p, g, m, v = pool
    n = 3 * 2 * sms() * 256 * 4 + 2
    s = State(p[:n], torch.zeros_like(g[:n]), torch.zeros_like(m[:n]), torch.zeros_like(v[:n]), lr=1e-2)
    gen = torch.Generator("cuda").manual_seed(9)
    for it in range(5):
        s.G.copy_(torch.randn(n, device="cuda", generator=gen) * 10.0 ** (-3 * it))
        s.lr.fill_(1e-2 / (it + 1))
        run_adam("carried step %d" % (it + 1), s, n, 0.9, 0.99, 1e-15, 0.5)
    assert int(s.step) == 5


def skip_pattern_state(n4, seed=3):
    """float4 groups by kind: 0, 1 all zero (skipped); 2 g = m = 0 with v != 0 (v still decays); 3, 4, 5 a single
    non-zero lane of v, m or g and nothing else; 6, 7 ordinary groups"""
    gen = torch.Generator("cuda").manual_seed(seed)
    p = torch.rand(n4, 4, device="cuda", generator=gen) * 2 - 1
    g = torch.randn(n4, 4, device="cuda", generator=gen) * 1e-3
    m = torch.randn(n4, 4, device="cuda", generator=gen) * 1e-3
    v = torch.rand(n4, 4, device="cuda", generator=gen) * 1e-6
    kind = (torch.arange(n4, device="cuda") % 8)[:, None]
    lane = (torch.arange(n4, device="cuda") // 8) % 4
    other = ~torch.nn.functional.one_hot(lane, 4).bool()  # the three lanes that stay zero in kinds 3-5
    g = torch.where((kind <= 4) | ((kind == 5) & other), 0.0, g)
    m = torch.where((kind <= 3) | (kind == 5) | ((kind == 4) & other), 0.0, m)
    v = torch.where((kind <= 1) | (kind == 4) | (kind == 5) | ((kind == 3) & other), 0.0, v)
    return tuple(x.reshape(-1).contiguous() for x in (p, g, m, v)), kind[:, 0]


def test_adam_skips_only_untouched_groups():
    n4 = 2 * sms() * 256 * 2 + 37
    (p, g, m, v), kind = skip_pattern_state(n4)
    n = 4 * n4 + 3  # the tail is never skipped
    s = State(*(torch.cat([x, torch.zeros(3, device="cuda")]) for x in (p, g, m, v)))
    before = s.clone()
    assert adam_step(s, n, 0.9, 0.999, 1e-15, 1.0) == 0
    torch.cuda.synchronize()
    check_call("skip patterns", before, s, n, 0.9, 0.999, 1e-15, 1.0, ph="skip")
    P1, V1, Ph1 = (x[:4 * n4].view(n4, 4) for x in (s.P, s.V, s.Ph))
    V0 = before.V[:4 * n4].view(n4, 4)
    skipped = kind <= 1
    assert torch.isnan(Ph1[skipped].float()).all(), "untouched groups must not be stored"
    assert not torch.isnan(Ph1[~skipped].float()).any(), "every other group must be stored"
    decays = kind == 2
    assert (V1[decays] < V0[decays]).all() and torch.equal(P1[decays], before.P[:4 * n4].view(n4, 4)[decays])
    assert not torch.isnan(s.Ph[4 * n4:].float()).any()


def test_adam_without_half_copy(pool):
    p, g, m, v = pool
    n = 2 * sms() * 256 * 4 + 6
    s = State(p[:n], g[:n], m[:n], v[:n], t=2)
    before = s.clone()
    assert adam_step(s, n, 0.9, 0.999, 1e-15, 1.0, ph=False) == 0
    torch.cuda.synchronize()
    check_call("params_half = NULL", before, s, n, 0.9, 0.999, 1e-15, 1.0, ph=None)
    assert torch.isnan(s.Ph.float()).all()


def test_adam_rejects_bad_arguments(pool):
    p, g, m, v = pool
    n = 64
    s = State(p[:n + 4], g[:n + 4], m[:n + 4], v[:n + 4], t=4)
    before = s.clone()
    L = _L()
    ptr = dict(P=s.P.data_ptr(), G=s.G.data_ptr(), M=s.M.data_ptr(), V=s.V.data_ptr(), Ph=s.Ph.data_ptr(),
               lr=s.lr.data_ptr(), step=s.step.data_ptr())

    def call(nn=n, inc=1, **over):
        a = dict(ptr, **over)
        return L.ngp_adam_step(a["P"], a["G"], a["M"], a["V"], a["Ph"], nn, a["lr"], a["step"], 0.9, 0.999, 1e-15, 1.0,
                               inc, _st())

    for k in ("P", "G", "M", "V", "lr", "step"):
        assert call(**{k: None}) == EINVAL, "NULL " + k
    for k in ("P", "G", "M", "V"):
        assert call(**{k: ptr[k] + 4}) == EINVAL, "misaligned " + k
    assert call(Ph=ptr["Ph"] + 2) == EINVAL, "misaligned params_half"
    assert call(nn=-1) == EINVAL
    torch.cuda.synchronize()
    for k, x in before.tensors().items():
        assert torch.equal(x.view(torch.uint8), getattr(s, k).view(torch.uint8)), k
    # n = 0: only the counter moves (and not even that without increment_step)
    assert call(nn=0, inc=0) == 0
    assert call(nn=0, inc=1) == 0
    torch.cuda.synchronize()
    assert int(s.step) == int(before.step) + 1
    for k in ("P", "G", "M", "V", "Ph"):
        assert torch.equal(getattr(before, k).view(torch.uint8), getattr(s, k).view(torch.uint8)), k
    # the exchange kernels: n must be a multiple of 4
    one = (C.c_uint64 * 1)
    flags = torch.zeros(64, dtype=torch.int32, device="cuda")
    sync = torch.zeros(8, dtype=torch.int32, device="cuda")
    assert L.ngp_adam_step_p2p(1, 0, one(ptr["G"]), ptr["P"], ptr["M"], ptr["V"], one(ptr["Ph"]), 6, ptr["lr"],
                               ptr["step"], 0.9, 0.999, 1e-15, 1, _st()) == EINVAL
    assert L.ngp_adam_step_fused(1, 0, one(ptr["G"]), one(ptr["Ph"]), one(flags.data_ptr()), 0, 0, ptr["P"], ptr["M"],
                                 ptr["V"], 6, None, sync.data_ptr(), ptr["lr"], ptr["step"], 0.9, 0.999, 1e-15, 1,
                                 _st()) == EINVAL


# ---- the exchange kernels with world = 1 ----------------------------------------------------------------------------
def exchange_state(pool, n, t):
    """random state with skip-pattern groups at the front; the fp16 copy equal to half(p), as the Trainer keeps it"""
    p, g, m, v = pool
    (ps, gs, ms, vs), _ = skip_pattern_state(4096)
    k = ps.numel()
    s = State(torch.cat([ps, p[:n - k]]), torch.cat([gs, g[:n - k]]), torch.cat([ms, m[:n - k]]),
              torch.cat([vs, v[:n - k]]), t=t)
    s.Ph = s.P.half()
    return s


def exchange_sizes():
    """fused: grid min(ceil(n4 / 1024), 3 SMs) of 256 threads, 4 groups per thread and trip at world 1: one partial trip,
    and several trips with a partial last one. p2p: grid min(ceil(n4 / 256), 4 SMs)"""
    return [4 * 4099, 4 * (2 * 3 * sms() * 1024 + 777)]


def fused_call(s, n, zero_buf, sync, flags, inc=1):
    one = (C.c_uint64 * 1)
    return _L().ngp_adam_step_fused(1, 0, one(s.G.data_ptr()), one(s.Ph.data_ptr()), one(flags.data_ptr()), 0, 0,
                                    s.P.data_ptr(), s.M.data_ptr(), s.V.data_ptr(), n, zero_buf.data_ptr(),
                                    sync.data_ptr(), s.lr.data_ptr(), s.step.data_ptr(), 0.9, 0.999, 1e-15, inc, _st())


def p2p_call(s, n, inc=1):
    one = (C.c_uint64 * 1)
    return _L().ngp_adam_step_p2p(1, 0, one(s.G.data_ptr()), s.P.data_ptr(), s.M.data_ptr(), s.V.data_ptr(),
                                  one(s.Ph.data_ptr()), n, s.lr.data_ptr(), s.step.data_ptr(), 0.9, 0.999, 1e-15, inc,
                                  _st())


def check_exchange(label, before, after, n):
    """within the bound, bitwise ngp_adam_step (grad_mul 1) on the same inputs, the consumed gradient untouched"""
    check_call(label, before, after, n, 0.9, 0.999, 1e-15, 1.0, ph="all", grad_cleared=False)
    assert torch.equal(after.G.view(torch.int32), before.G.view(torch.int32)), label + ": consumed gradient changed"
    ref = before.clone()
    assert adam_step(ref, n, 0.9, 0.999, 1e-15, 1.0) == 0
    torch.cuda.synchronize()
    for k in ("P", "M", "V"):
        assert torch.equal(getattr(ref, k).view(torch.int32), getattr(after, k).view(torch.int32)), label + ": " + k
    assert torch.equal(ref.Ph.view(torch.int16), after.Ph.view(torch.int16)), label + ": Ph"
    assert torch.equal(ref.step, after.step)


@pytest.mark.parametrize("n_idx", [0, 1])
def test_fused_exchange_world1(pool, n_idx):
    n = exchange_sizes()[n_idx]
    s = exchange_state(pool, n, t=2)
    flags = torch.zeros(64, dtype=torch.int32, device="cuda")
    sync = torch.zeros(8, dtype=torch.int32, device="cuda")
    zero_buf = torch.ones(n, device="cuda")
    for call in range(1, 4):
        s.lr.fill_(1e-2 / call)
        before = s.clone()
        zero_buf.fill_(1.0)
        assert fused_call(s, n, zero_buf, sync, flags) == 0
        torch.cuda.synchronize()
        check_exchange("fused n=%d call %d" % (n, call), before, s, n)
        assert zero_buf.abs().max().item() == 0, "zero_buf must be cleared"
        assert int(sync[0]) == call and int(flags[0]) == call and int(flags[16]) == call, (sync.tolist(), flags.tolist())
        assert int(sync[1]) == 0 and int(sync[2]) == 0 and int(sync[3]) == call
        s.G.copy_(torch.randn(n, device="cuda", generator=torch.Generator("cuda").manual_seed(call)) * 1e-3)


def test_fused_exchange_world1_graph_replays(pool):
    n = exchange_sizes()[1]
    s = exchange_state(pool, n, t=1)
    flags = torch.zeros(64, dtype=torch.int32, device="cuda")
    sync = torch.zeros(8, dtype=torch.int32, device="cuda")
    zero_buf = torch.ones(n, device="cuda")
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        assert fused_call(s, n, zero_buf, sync, flags) == 0
    torch.cuda.synchronize()
    assert int(s.step) == 0 and int(sync[0]) == 0, "capturing must not run the kernel"
    for replay in range(1, 4):
        before = s.clone()
        zero_buf.fill_(1.0)
        graph.replay()
        torch.cuda.synchronize()
        check_exchange("fused graph replay %d" % replay, before, s, n)
        assert zero_buf.abs().max().item() == 0
        assert int(sync[0]) == replay and int(flags[0]) == replay and int(flags[16]) == replay
        assert int(sync[2]) == 0 and int(s.step) == replay


@pytest.mark.parametrize("n_idx", [0, 1])
def test_p2p_exchange_world1(pool, n_idx):
    n = exchange_sizes()[n_idx]
    s = exchange_state(pool, n, t=3)
    for call in range(1, 3):
        before = s.clone()
        assert p2p_call(s, n) == 0
        torch.cuda.synchronize()
        check_exchange("p2p n=%d call %d" % (n, call), before, s, n)


# ---- the Trainer's wiring -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("schedule", [False, True])
def test_trainer_step_matches_float64(schedule):
    """a captured single-GPU Trainer on the Lego scene; the after_backward hook snapshots G, P, M, V, lr and the counter;
    P, M and V after the step are within the bound of the float64 step from that snapshot (betas in order, eps,
    grad_mul = 1 / world, t = step + 1). Steps 1, 2, 3 -- or step 30 under CosineAnnealingLR"""
    from ngp_pl_b200 import synth
    from ngp_pl_b200.models.networks import NGP
    from ngp_pl_b200.trainer import CosineAnnealingLR, Trainer
    torch.manual_seed(0)
    scene = synth.lego_scene(0)
    model = NGP(scene.scale).cuda()
    bank = synth.RayBank(scene, n_images=8, device="cuda", seed=3)
    sched = CosineAnnealingLR(1e-2, T_max=8, steps_per_epoch=4) if schedule else None
    tr = Trainer(model, n_rays=4096, lr_schedule=sched)
    assert tr.n_params == 11455280
    tr.attach_bank(bank)
    tr.capture(sample=True)
    check_at = {30} if schedule else {1, 2, 3}
    snap = {}

    def hook(t_):
        snap.update(G=t_.G.clone(), P=t_.P.clone(), M=t_.M.clone(), V=t_.V.clone(), lr=t_.lr_dev.clone(),
                    step=t_.step_dev.clone())

    for k in range(1, max(check_at) + 1):
        tr.train_step(after_backward=hook if k in check_at else None)
        if k not in check_at:
            continue
        torch.cuda.synchronize()
        t = int(snap["step"]) + 1
        assert t == k and int(tr.step_dev) == k
        lr = float(snap["lr"])
        if schedule:
            assert lr == A.f32(sched.lr_at_step(k - 1)) and lr != A.f32(1e-2)
        assert snap["G"].abs().max() > 0
        o = A.step(snap["P"], snap["G"], snap["M"], snap["V"], t, lr, tr.betas[0], tr.betas[1], tr.eps,
                   1.0 / tr.world_size, m_k=tr.M, v_k=tr.V)
        note("trainer m'", A.ratio(tr.M.double() - o["m"], o["m_err"]))
        note("trainer v'", A.ratio(tr.V.double() - o["v"], o["v_err"]))
        rp = A.ratio(tr.P.double() - o["p"], o["p_err"])
        WORST_P[(A.f32(tr.betas[1]), t)] = max(WORST_P.get((A.f32(tr.betas[1]), t), 0.0), rp)
        note("trainer p'", rp)
        assert torch.equal(tr.Ph.view(torch.int16), tr.P.half().view(torch.int16))
        assert tr.G.abs().max().item() == 0
