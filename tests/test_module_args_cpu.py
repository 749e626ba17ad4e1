"""Argument checks of the stand-alone module backward entry points (ngp_mlp_rgb_backward, ngp_enc_backward).

Their kernels read x_half as uint32 words, dL_dh as float2 and feat_save as uint4, so a misaligned pointer must be
refused with NGP_EINVAL before the call touches the device. The pointers below are fake addresses that nothing may
dereference: every call must return at its argument checks, which also makes this test run without a GPU.
"""
import ctypes as C

import numpy as np
import pytest

NGP_EINVAL = -22
P = 1 << 24  # a fake, 256-byte aligned address
N = 37       # rows: more than one 16-row tile, not a multiple of 16


@pytest.fixture(scope="module")
def L():
    from ngp_pl_b200 import _lib
    return _lib.lib()


def _rgb_bwd(L, x_half=P, dL_dx=P):
    # (rgb_params_h, x_half, dL_dout3, n, rgb_act, loss_scale, dL_dx, grad_rgb, stream)
    return L.ngp_mlp_rgb_backward(P, x_half, P, N, 1, P, dL_dx, P, None)


@pytest.mark.parametrize("offset", [1, 2, 3])
def test_mlp_rgb_backward_refuses_misaligned_input(L, offset):
    assert _rgb_bwd(L, x_half=P + offset) == NGP_EINVAL


@pytest.mark.parametrize("offset", [4])
def test_mlp_rgb_backward_refuses_misaligned_input_gradient(L, offset):
    assert _rgb_bwd(L, dL_dx=P + offset) == NGP_EINVAL


def _enc_bwd(L, dL_dh=P, feat_save=P, n_levels=16):
    from ngp_pl_b200 import _lib
    L_ = min(max(n_levels, 1), 16)
    meta, _ = _lib.grid_meta(L_, 19, 16, float(np.exp(np.log(2048 * 0.5 / 16) / max(L_ - 1, 1))))
    meta.n_levels = n_levels
    net = _lib.NgpNet()
    net.enc_params_h = P
    net.rgb_params_h = None
    net.meta = meta
    for k in range(3):
        net.xyz_min[k], net.xyz_max[k] = 0.0, 1.0
    net.rgb_act = 1
    smp = _lib.NgpSamples()
    smp.xyzs = P
    smp.dirs = smp.rays_o = smp.rays_d = smp.ray_idx = smp.ts = None
    smp.n = N
    ws = L.ngp_net_backward_workspace(N)
    # (net, smp, dL_dh, feat_save, loss_scale, grad_enc, workspace, workspace_bytes, stream)
    return L.ngp_enc_backward(C.byref(net), C.byref(smp), dL_dh, feat_save, P, P, P, ws, None)


@pytest.mark.parametrize("offset", [2, 4])
def test_enc_backward_refuses_misaligned_output_gradient(L, offset):
    assert _enc_bwd(L, dL_dh=P + offset) == NGP_EINVAL


@pytest.mark.parametrize("offset", [4, 8])
def test_enc_backward_refuses_misaligned_saved_features(L, offset):
    assert _enc_bwd(L, feat_save=P + offset) == NGP_EINVAL


@pytest.mark.parametrize("n_levels", [0, 17])
def test_enc_backward_refuses_level_count_out_of_range(L, n_levels):
    assert _enc_bwd(L, n_levels=n_levels) == NGP_EINVAL
