"""The float64 backward reference (oracle/grad64.py) against the existing restatements, so that a wrong reference cannot
silently agree with a wrong kernel (tests/test_backward_fp64_gpu.py compares the kernels with it):
  * its network backward against fp32 autograd of oracle.torch_ngp_forward (rgb_act 0 and 1);
  * its table scatter against float64 autograd of oracle.torch_grid_encode (dense, hashed and wrapping corners);
  * its feat_save decoder against a plain encoder of the documented fragment layout.
"""
import numpy as np
import pytest
import torch

from oracle import grad64


def _points(n, seed, lo=-0.5, hi=0.5):
    rng = np.random.RandomState(seed)
    x = rng.uniform(lo, hi, (n, 3)).astype(np.float32)
    d = (rng.normal(size=(n, 3)) * rng.uniform(0.5, 2.0, (n, 1))).astype(np.float32)
    return torch.as_tensor(x), torch.as_tensor(d)


def _params(meta_total, seed, table_amp=0.5):
    """the modules' initialisation (ngp_pl_b200/tcnn.py) with an O(1) table, so every level matters"""
    g = torch.Generator().manual_seed(seed)
    enc = torch.empty(3072 + 2 * meta_total)
    enc[:2048].uniform_(-(6 / 96) ** 0.5, (6 / 96) ** 0.5, generator=g)
    enc[2048:3072].uniform_(-(6 / 80) ** 0.5, (6 / 80) ** 0.5, generator=g)
    enc[3072:].uniform_(-table_amp, table_amp, generator=g)
    rgb = torch.empty(7168)
    rgb[:2048].uniform_(-(6 / 96) ** 0.5, (6 / 96) ** 0.5, generator=g)
    rgb[2048:6144].uniform_(-(6 / 128) ** 0.5, (6 / 128) ** 0.5, generator=g)
    rgb[6144:].uniform_(-(6 / 80) ** 0.5, (6 / 80) ** 0.5, generator=g)
    return enc.half().float(), rgb.half().float()  # fp16-representable masters: the fp16 working copy is exact


@pytest.mark.parametrize("rgb_act", [1, 0])
def test_reference_chain_vs_fp32_autograd(oracle, rgb_act):
    meta, total = oracle.grid_meta(16, 19, 16, float(np.float32(np.exp(np.log(2048 * 0.5 / 16) / 15))))
    enc, rgb = _params(total, 7)
    n = 300
    x, d = _points(n, 3)
    mn, mx = torch.full((1, 3), -0.5), torch.full((1, 3), 0.5)
    x01 = (x - mn) / (mx - mn)
    with torch.no_grad():
        feat = oracle.torch_grid_encode(meta, enc[3072:].view(-1, 2), x01).half()
    rng = np.random.RandomState(4)
    up_sig = torch.as_tensor((rng.normal(size=n) * 1e-2).astype(np.float32))
    up_rgb = torch.as_tensor((rng.normal(size=(n, 3)) * 1e-1).astype(np.float32))
    scale = 2.0 ** 10
    ref = grad64.mlp_backward(feat, grad64.sh4_64(d), enc[:3072], rgb, up_sig, up_rgb, scale, rgb_act)
    # rows whose ReLU masks the reference cannot pin down take no part (their branch may legitimately differ)
    keep = ~ref["ambiguous"]
    assert keep.sum() >= n - 3
    up_sig, up_rgb = up_sig * keep, up_rgb * keep[:, None]
    ref = grad64.mlp_backward(feat, grad64.sh4_64(d), enc[:3072], rgb, up_sig, up_rgb, scale, rgb_act)

    e, r = enc.clone().requires_grad_(True), rgb.clone().requires_grad_(True)
    sig, out, _ = oracle.torch_ngp_forward(meta, e, r, mn, mx, x, d, rgb_act=rgb_act)
    ((sig * up_sig).sum() + (out * up_rgb).sum()).backward()
    # autograd differentiates the sigmoid at its unrounded value o' = sigmoid(y), the kernel at o = fp16(o'):
    # |o' (1 - o') - o (1 - o)| <= 2^-11 o, i.e. 2^-11 o / (1 - o) of the out-gradient, carried linearly down the chain
    kappa = 0.0
    if rgb_act == 1:
        o = ref["o"]
        kappa = 2.0 ** -11 * float((o / (1 - o)).max())
    got = grad64.split_dW(e.grad.double(), r.grad.double())
    for k, (v, A, err) in ref["dW"].items():
        # the reference is an fp16-rounded chain, autograd an unrounded fp32 one: they differ by at most the reference's own
        # rounding bound, plus fp32 accumulation (2^-18 A) and the sigmoid term
        tol = err + (2.0 ** -18 + kappa) * A
        assert (got[k] - v).abs().le(tol).all(), "%s: max excess %g" % (k, float(((got[k] - v).abs() - tol).max()))
        assert v.abs().max() > 0
    # the table gradient: the reference's dfeat scattered, against autograd through the fp32 grid encoding
    tg, S, _ = grad64.grid_scatter(meta, x01, ref["dfeat"], 1.0 / scale, total)
    terr, _, _ = grad64.grid_scatter(meta, x01, ref["dfeat_err"] + kappa * ref["dfeat_abs"], 1.0 / scale, total)
    ag = e.grad[3072:].double().view(-1, 2)
    tol = terr + 2.0 ** -18 * grad64.grid_scatter(meta, x01, ref["dfeat_abs"], 1.0 / scale, total)[0] + 1e-30
    assert (ag - tg).abs().le(tol + 2.0 ** -20 * S).all()
    assert tg.abs().max() > 0


@pytest.mark.parametrize("cfg", [(16, 19), (4, 14)])
def test_reference_scatter_vs_float64_autograd(oracle, cfg):
    L, log2_T = cfg
    meta, total = oracle.grid_meta(L, log2_T, 16, float(np.float32(np.exp(np.log(2048 * 0.5 / 16) / 15))))
    assert meta.hashed_mask != 0 and meta.hashed_mask != (1 << L) - 1  # dense and hashed levels both present
    n = 400
    rng = np.random.RandomState(11)
    x01 = rng.uniform(0, 1, (n, 3)).astype(np.float32)
    # upper wrap of the dense levels, the last float below 1, and exact grid vertices of the finest dense level
    x01[:6] = [[1, 1, 1], [0, 0, 0], [1, 0, 1], [1 - 2 ** -24] * 3, [1, 1 - 2 ** -24, 0.5], [0.5, 0.25, 1]]
    l_dense = max(l for l in range(L) if not (meta.hashed_mask >> l) & 1)
    x01[6:20] = (rng.randint(0, int(meta.res[l_dense]), (14, 3)) / np.float32(meta.scale[l_dense])).astype(np.float32)
    x01 = torch.as_tensor(np.clip(x01, 0, 1))
    G = torch.as_tensor(rng.normal(size=(n, 32)).astype(np.float16)).double()
    G[:, 2 * L:] = 0
    table = torch.zeros(total, 2, dtype=torch.float64, requires_grad=True)
    feat = oracle.torch_grid_encode(meta, table, x01)
    (feat * G).sum().backward()
    ref, S, m = grad64.grid_scatter(meta, x01, G.half(), 1.0, total)
    assert (table.grad - ref).abs().le(1e-6 * S).all()
    assert int(m.sum()) == 8 * L * n and (ref != 0).sum() > 0


def _encode_np(feat):
    """feat (n, 32) float16 -> bytes of the fragment layout, written element by element from its description"""
    n = feat.shape[0]
    t = (n + 31) // 32 * 2
    out = np.zeros((t, 2, 32, 4, 2), np.float16)  # tile, kt, lane, word, half
    for row in range(n):
        tile, r = divmod(row, 16)
        g, rh = r % 8, r // 8
        for col in range(32):
            kt, c = divmod(col, 16)
            ch, cc = divmod(c, 8)
            q, half = divmod(cc, 2)
            word = 2 * ch + rh  # x: (g, 2q) y: (g + 8, 2q) z: (g, 2q + 8) w: (g + 8, 2q + 8)
            out[tile, kt, 4 * g + q, word, half] = feat[row, col]
    return out.tobytes()


def test_feat_save_decoder_vs_fragment_layout():
    rng = np.random.RandomState(5)
    for n in (1, 16, 37, 64):
        feat = rng.normal(size=(n, 32)).astype(np.float16)
        raw = torch.frombuffer(bytearray(_encode_np(feat)), dtype=torch.uint8)
        assert torch.equal(grad64.decode_feat_save(raw, n), torch.as_tensor(feat))
        assert torch.equal(grad64.encode_feat_save(torch.as_tensor(feat)), raw)
    # column 2 l (+1) is level l: level q lives in lane q's words x / y of k-tile 0
    raw = np.zeros(2 * 1024, np.uint8).view(np.float16)
    raw.reshape(2, 2, 32, 4, 2)[0, 0, 4 * 3 + 1, 1, 0] = 1.0  # tile 0, kt 0, g = 3, q = 1, word y (row g + 8), low half
    dec = grad64.decode_feat_save(torch.as_tensor(raw.view(np.uint8)), 16)
    assert dec[11, 2].item() == 1.0 and dec.abs().sum().item() == 1.0
