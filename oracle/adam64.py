"""float64 restatement of one Adam step as the optimiser kernels take it, with a bound on how far their fp32 results may
lie from it -- TEST INFRASTRUCTURE ONLY.

Nothing under ngp_pl_b200/ imports this. It is plain torch on any device: the GPU tests run it on CUDA at the Trainer's
11.4 M parameters, the CPU suite holds it to exact rational arithmetic, to torch.optim.Adam and to a float32 replay of
the kernels' expression order (tests/test_adam64_cpu.py).

Semantics: apex FusedAdam as the reference builds it (train.py:131: adam_w_mode, bias correction on, weight decay 0),
on the fp32 inputs the kernels read. beta1, beta2, eps, lr and grad_mul are the float32 values the kernels receive;
t = (the device step counter) + 1.
    g  = grad * grad_mul
    m' = beta1 m + (1 - beta1) g
    v' = beta2 v + (1 - beta2) g^2
    p' = p - lr (m' / bc1) / (sqrt(v' / bc2) + eps),   bc = 1 - beta^t in float64 (apex: 1 - std::pow(beta, step) in
                                                        double, rounded to float once)
m' and v' are computed from the kernel's inputs; p' from the kernel's own stored m' and v' (`m_k`, `v_k`), so that the
bound on p' does not carry the moments' roundings twice.

The bounds (`*_err`) are first order in the fp32 unit roundoff u = 2^-24, with an absolute 2^-150 (half the smallest
subnormal) for every rounding that can land in the subnormal range: the build has no -ftz, and v of a hash entry with a
tiny gradient is subnormal. Tests compare with SAFETY (= 2) times the bound. Step by step, as the kernels compute:
  * g = fl(grad grad_mul): u |g| (0 when grad_mul is a power of two, up to the subnormal term).
  * 1 - beta: exact for beta in [0.5, 1] (Sterbenz); otherwise its own rounding, carried.
  * m' = fl(beta1 m + fl((1 - beta1) g)): u (|beta1 m| + |(1 - beta1) g|) + u |m'| -- with or without the fma
    contraction -- plus (1 - beta1) |dg|.
  * v' = beta2 v + fl(fl((1 - beta2) g) g): 2 u |(1 - beta2) g^2| + u |beta2 v| + u |v'| plus 2 (1 - beta2) |g dg|.
  * step_size = fl(lr / fl(bc1)): 2 u.  inv_sqrt_bc2 = rsqrtf(fl(bc2)): u / 2 from bc2, 2 ulp (CUDA's documented
    rsqrtf error) = 4 u.  bc1 and bc2 are allowed ONE float rounding of the float64 value each, apex's accuracy: a
    kernel that forms 1 - powf(beta, t) in float loses up to ~100 u of bc2 to cancellation at small t (beta2 = 0.999),
    and the bound does not absorb that.
  * q = fl(fl(sqrt(v')) inv_sqrt_bc2): u (IEEE sqrtf) + u (product) + the constant's error; D = fl(q + eps): + u D;
    Q = fl(m' / D): |Q| dD / D + u |Q|; the update S Q: |Q| dS + S dQ + u |S Q|.
  * p' = fl(p - S Q): the update's error plus half an ulp of the result (of the binade that holds |p'| + the update's
    error, which contains the exact difference).
"""
import math

import torch

U = 2.0 ** -24       # fp32 unit roundoff (round to nearest)
ULP = 2.0 ** -23     # one fp32 ulp relative to the value it is measured at (upper bound over a binade)
TINY = 2.0 ** -150   # largest error of one rounding into the subnormal range (half the smallest subnormal)
RSQRT_ULP = 2.0      # CUDA's documented maximum error of rsqrtf
SAFETY = 2.0         # the tests compare with SAFETY * bound: second-order terms of the first-order bound


def f32(x):
    """the float32 value a float argument is rounded to when the kernel receives it, as a Python float"""
    return float(torch.tensor(float(x), dtype=torch.float32))


def bias_correction(beta, t):
    """1 - beta^t of the float32 beta, in float64 (apex's host computation before its single rounding to float)"""
    return -math.expm1(t * math.log(f32(beta)))


def bias_correction_apex(beta, t):
    """apex's recipe: 1 - pow(double(beta), t) rounded to float once (what the kernels compute)"""
    return f32(1.0 - math.pow(f32(beta), t))


def half_ulp(x):
    """half an fp32 ulp of the binade holding |x| (>= 2^-150: the subnormal spacing), float64 tensor"""
    x = x.abs()
    # fl32(x) in [2^(e-1), 2^e): ulp = 2^(e-24). Rounding is monotone and powers of two are floats, so fl32(x)'s binade
    # is never below x's own
    _, e = torch.frexp(x.to(torch.float32).clamp_min(2.0 ** -126))
    return torch.ldexp(torch.ones_like(x), (e - 25).to(x.dtype)).clamp_min(TINY)


def step(p, g, m, v, t, lr, beta1, beta2, eps, grad_mul=1.0, m_k=None, v_k=None):
    """One Adam step of fp32 tensors p, g, m, v (any device), in float64. t: the step the kernel takes (counter + 1),
    lr / betas / eps / grad_mul as passed to the kernel (rounded to float32 here). m_k, v_k: the kernel's stored
    m' and v', from which p' is computed (default: float64's own). Returns m, m_err, v, v_err, p, p_err."""
    assert t >= 1
    d = torch.float64
    b1, b2, eps, lr, gm = f32(beta1), f32(beta2), f32(eps), f32(lr), f32(grad_mul)
    c1, c2 = 1.0 - b1, 1.0 - b2
    dc1, dc2 = abs(f32(c1) - c1), abs(f32(c2) - c2)  # 0 for beta >= 0.5
    p, g, m, v = p.to(d), g.to(d), m.to(d), v.to(d)

    gr = g * gm
    gr_err = U * gr.abs() + TINY
    if math.frexp(gm)[0] == 0.5:  # a power of two: exact unless the product is subnormal
        gr_err = torch.where(gr.abs() < 2.0 ** -126, TINY, 0.0)

    m1 = b1 * m + c1 * gr
    m1_err = c1 * gr_err + dc1 * gr.abs() + U * ((b1 * m).abs() + (c1 * gr).abs()) + U * m1.abs() + 4 * TINY
    v1 = b2 * v + c2 * gr * gr
    v1_err = 2 * c2 * gr.abs() * gr_err + dc2 * gr * gr + 2 * U * c2 * gr * gr + U * (b2 * v).abs() + U * v1 + 5 * TINY

    mk = m1 if m_k is None else m_k.to(d)
    vk = v1 if v_k is None else v_k.to(d)
    bc1, bc2 = bias_correction(beta1, t), bias_correction(beta2, t)
    S = lr / bc1
    dS = 2 * U * S
    R = 1.0 / math.sqrt(bc2)
    dR = (U / 2 + RSQRT_ULP * ULP) * R
    s = torch.sqrt(vk)
    q = s * R
    dq = U * q + s * dR + U * q
    D = q + eps
    dD = dq + U * D
    Q = mk / D
    dQ = Q.abs() * dD / D + U * Q.abs() + TINY
    upd = S * Q
    dupd = dS * Q.abs() + S * dQ + U * upd.abs() + TINY
    p1 = p - upd
    p1_err = dupd + half_ulp(p1.abs() + dupd)
    return dict(m=m1, m_err=m1_err, v=v1, v_err=v1_err, p=p1, p_err=p1_err, update=upd, update_err=dupd)


def _log_uniform(gen, n, lo, hi):
    x = torch.rand(n, generator=gen, dtype=torch.float64) * (math.log(hi) - math.log(lo)) + math.log(lo)
    sign = torch.where(torch.rand(n, generator=gen) < 0.5, -1.0, 1.0).double()
    return sign * x.exp()


def random_state(n, seed):
    """fp32 (p, g, m, v) on the CPU over the ranges the optimiser meets and beyond: gradients 1e-25 .. 1e4 (v' subnormal
    or 0 at the low end), moments unrelated to them, parameters from O(1) down to the hash table's 1e-4 initialisation
    and below (there the update, not p's own rounding, dominates p'), and exact zeros in each"""
    gen = torch.Generator().manual_seed(seed)
    g = _log_uniform(gen, n, 1e-25, 1e4)
    m = _log_uniform(gen, n, 1e-30, 1e2)
    v = _log_uniform(gen, n, 1e-44, 1e6).abs()
    p = torch.where(torch.rand(n, generator=gen) < 0.5, torch.rand(n, generator=gen, dtype=torch.float64) * 2 - 1,
                    _log_uniform(gen, n, 1e-8, 1e-2))
    for x in (g, m, v, p):
        x[torch.rand(n, generator=gen) < 0.05] = 0.0
    return tuple(x.float() for x in (p, g, m, v))


def ratio(err, bound):
    """largest |err| / (SAFETY bound) (0 where both are 0; inf where the bound is 0 and err is not)"""
    err, bound = err.double().abs(), SAFETY * bound.double()
    r = torch.where(bound > 0, err / bound.clamp_min(1e-300), torch.where(err > 0, math.inf, 0.0))
    return float(r.max()) if r.numel() else 0.0
