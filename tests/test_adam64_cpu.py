"""The float64 Adam restatement oracle/adam64.py and its bound, without a GPU: against exact rational arithmetic, against
torch.optim.Adam in float64, and against a float32 replay of the optimiser kernels' expression order -- which the bound
must contain when the bias corrections are computed as apex computes them, and must NOT contain when they are formed in
float (1 - powf(beta, t)), whose cancellation at small t is the error the GPU test is there to catch."""
import math
from fractions import Fraction

import numpy as np
import pytest
import torch

from oracle import adam64 as A

T_ALL = (1, 2, 3, 5, 10, 100, 1000, 10 ** 4, 10 ** 5)
BETAS = ((0.9, 0.999), (0.9, 0.99), (0.5, 0.75))


def _frac_sqrt(x, bits=200):
    """sqrt of a non-negative Fraction to within a relative 2^-bits"""
    if x == 0:
        return Fraction(0)
    a, b = x.numerator, x.denominator
    return Fraction(math.isqrt(a * b * 4 ** bits), b * 2 ** bits)


def _exact_step(p, g, m, v, t, lr, beta1, beta2, eps, grad_mul):
    F = Fraction
    b1, b2, lr, eps, gm = (F(A.f32(x)) for x in (beta1, beta2, lr, eps, grad_mul))
    gr = F(g) * gm
    m1 = b1 * F(m) + (1 - b1) * gr
    v1 = b2 * F(v) + (1 - b2) * gr * gr
    bc1, bc2 = 1 - b1 ** t, 1 - b2 ** t
    p1 = F(p) - lr * (m1 / bc1) / (_frac_sqrt(v1 / bc2) + eps)
    return m1, v1, p1


def _constructed():
    """m = 0 with v != 0, g = 0 with m != 0, all zero, a subnormal v, g alone, and opposite signs"""
    rows = [(0.5, 1e-3, 0.0, 4e-6), (0.25, 0.0, -2e-3, 1e-6), (-1e-4, 0.0, 0.0, 0.0), (1e-4, 0.0, 0.0, 3e-40),
            (0.0, 2e-20, 0.0, 0.0), (3e-5, -7.0, 0.5, 20.0), (1.0, 1e4, -1e2, 1e6), (-0.75, 1e-25, 1e-30, 1e-44)]
    return [tuple(float(np.float32(x)) for x in r) for r in rows]


@pytest.mark.parametrize("t", (1, 2, 3, 10, 100, 1000))
@pytest.mark.parametrize("betas", BETAS)
def test_restatement_matches_exact_arithmetic(t, betas):
    b1, b2 = betas
    eps, lr, gm = 1e-8, 1e-2, 1.0 / 3
    p, g, m, v = A.random_state(300, seed=t)
    rows = _constructed() + list(zip(p.tolist(), g.tolist(), m.tolist(), v.tolist()))
    pt, gt, mt, vt = (torch.tensor([r[k] for r in rows], dtype=torch.float32) for k in range(4))
    o = A.step(pt, gt, mt, vt, t, lr, b1, b2, eps, gm)
    assert A.bias_correction(b2, t) == pytest.approx(float(1 - Fraction(A.f32(b2)) ** t), rel=1e-15)
    for i, (pi, gi, mi, vi) in enumerate(rows):
        m1, v1, p1 = _exact_step(pi, gi, mi, vi, t, lr, b1, b2, eps, gm)
        gr = abs(gi * A.f32(gm))
        # relative to the sum of the magnitudes the float64 value was formed from (its terms may cancel)
        for name, want, size in (("m", m1, abs(A.f32(b1) * mi) + gr), ("v", v1, vi + gr * gr),
                                 ("p", p1, abs(pi) + abs(float(p1) - pi))):
            got = float(o[name][i])
            assert abs(Fraction(got) - want) <= Fraction(1e-15 * size) + Fraction(1, 2 ** 1070), (name, i, got, float(want))
    # the constructed rows: m' = 0 gives p' = p exactly; g = 0 still moves p with the momentum
    assert float(o["p"][0]) != rows[0][0] and float(o["p"][2]) == rows[2][0] and float(o["p"][1]) > rows[1][0]


@pytest.mark.parametrize("betas", BETAS)
def test_restatement_matches_torch_adam(betas):
    """torch.optim.Adam in float64 with the float32-rounded hyper-parameters, five steps, per-step gradients"""
    b1, b2 = (A.f32(b) for b in betas)
    lr, eps = A.f32(1e-2), A.f32(1e-15)
    p, _, _, _ = A.random_state(20000, seed=7)
    ref = p.double().clone().requires_grad_(True)
    opt = torch.optim.Adam([ref], lr=lr, betas=(b1, b2), eps=eps, foreach=False)
    P, M, V = p.double(), torch.zeros(p.numel(), dtype=torch.float64), torch.zeros(p.numel(), dtype=torch.float64)
    gen = torch.Generator().manual_seed(3)
    for t in range(1, 6):
        g = (torch.randn(p.numel(), generator=gen, dtype=torch.float64) * 10.0 ** (2 - t)).float().double()
        ref.grad = g.clone()
        opt.step()
        o = A.step(P, g, M, V, t, lr, b1, b2, eps, 1.0)  # float64 state in, float64 throughout
        st = opt.state[ref]
        # relative to the magnitudes each value is formed from (m's two terms may cancel, and p's with the update).
        # torch forms 1 - beta^t in double, which cancels like the float version does: its bias corrections carry up
        # to 2^-53 beta^t / (1 - beta^t), which reaches the update (bc2 through a square root)
        bc1, bc2 = A.bias_correction(b1, t), A.bias_correction(b2, t)
        mag = b1 * M.abs() + (1 - b1) * g.abs()
        upd_mag = lr / bc1 * mag / ((o["v"] / bc2).sqrt() + eps)
        upd_rel = 2.0 ** -52 * (4 + b1 ** t / bc1 + 0.5 * b2 ** t / bc2)
        assert ((o["m"] - st["exp_avg"]).abs() <= 1e-15 * mag).all(), t
        assert ((o["v"] - st["exp_avg_sq"]).abs() <= 1e-15 * o["v"]).all(), t
        assert ((o["p"] - ref.detach()).abs() <= 2.0 ** -52 * P.abs() + upd_rel * upd_mag).all(), t
        P, M, V = ref.detach().clone(), st["exp_avg"].clone(), st["exp_avg_sq"].clone()


def replay_f32(p, g, m, v, t, lr, beta1, beta2, eps, grad_mul, float_power=False):
    """the kernels' expression order in numpy float32 (no fma; numpy keeps subnormals): g * grad_mul, the moments,
    step_size = lr / bc1, rsqrt(bc2) correctly rounded, sqrt(v') * rsqrt + eps, m' / denom, p - step_size * that"""
    f = np.float32
    b1, b2, lr, eps, gm = f(beta1), f(beta2), f(lr), f(eps), f(grad_mul)
    if float_power:
        bc1, bc2 = f(1) - np.power(b1, f(t)), f(1) - np.power(b2, f(t))
    else:
        bc1, bc2 = f(A.bias_correction_apex(beta1, t)), f(A.bias_correction_apex(beta2, t))
    step_size = f(lr / bc1)
    inv = f(1.0 / math.sqrt(float(bc2)))
    with np.errstate(under="ignore"):
        gr = g * gm
        m1 = b1 * m + (f(1) - b1) * gr
        v1 = b2 * v + (f(1) - b2) * gr * gr
        denom = np.sqrt(v1) * inv + eps
        p1 = p - step_size * (m1 / denom)
    return p1, m1, v1


def _replay_ratios(state, t, betas, eps, gm, float_power):
    p, g, m, v = state
    p1, m1, v1 = replay_f32(p.numpy(), g.numpy(), m.numpy(), v.numpy(), t, 1e-2, betas[0], betas[1], eps, gm,
                            float_power)
    assert p1.dtype == np.float32 and m1.dtype == np.float32 and v1.dtype == np.float32
    o = A.step(p, g, m, v, t, 1e-2, betas[0], betas[1], eps, gm, m_k=torch.from_numpy(m1), v_k=torch.from_numpy(v1))
    return {k: A.ratio(torch.from_numpy(x).double() - o[k], o[k + "_err"])
            for k, x in (("m", m1), ("v", v1), ("p", p1))}


@pytest.fixture(scope="module")
def state():
    return A.random_state(10 ** 6, seed=11)


@pytest.mark.parametrize("t", T_ALL)
def test_float32_replay_within_bound(state, t):
    """10^6 elements, every beta pair, eps 1e-15 and 1e-8, grad_mul 1, 1/2, 1/3: the apex-style replay lies within the bound"""
    worst = {}
    for betas in BETAS:
        for eps in (1e-15, 1e-8):
            for gm in (1.0, 0.5, 1.0 / 3):
                r = _replay_ratios(state, t, betas, eps, gm, float_power=False)
                for k in r:
                    worst[k] = max(worst.get(k, 0.0), r[k])
    print("t=%d: replay error / (2 x bound): %s" % (t, {k: round(x, 3) for k, x in worst.items()}))
    assert all(x <= 1.0 for x in worst.values()), worst


@pytest.mark.parametrize("t", (2, 3, 5))
def test_float_power_bias_correction_falls_outside_bound(state, t):
    """1 - powf(0.999, t) in float: the cancellation moves p' beyond the bound at small t; beta1's is harmless"""
    r = _replay_ratios(state, t, (0.9, 0.999), 1e-15, 1.0, float_power=True)
    print("t=%d, float bias corrections: %s" % (t, r))
    assert r["p"] > 1.4, r
    assert r["m"] <= 1.0 and r["v"] <= 1.0
