"""Gather and mean logic of metrics.evaluate on CPU: two `gloo` processes (world_size 2, 127.0.0.1), each holding the
per-view rows of its shard_range of the views, must report what one rank holding every view reports, in view order."""
import math
import os
import socket

import torch
import torch.distributed as dist
import torch.multiprocessing as mp

N_VIEWS, N_PIX = 7, 800 * 600  # 7 views: shards of 4 and 3


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _rows():
    """[sum of squared errors, SSIM, total_samples] per view; view 5 is a perfect render (PSNR +inf)"""
    g = torch.Generator().manual_seed(11)
    rows = torch.stack([torch.rand(N_VIEWS, generator=g, dtype=torch.float64) * 3 * N_PIX * 1e-3,
                        torch.rand(N_VIEWS, generator=g, dtype=torch.float64),
                        torch.randint(1, 1 << 40, (N_VIEWS,), generator=g).double()], 1)
    rows[5, 0] = 0.0
    return rows


def _worker(rank, world, port, out):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from ngp_pl_b200.metrics import gather_metrics
    from ngp_pl_b200.trainer import shard_range
    lo, hi = shard_range(N_VIEWS, world, rank)
    res = gather_metrics(_rows()[lo:hi].clone(), N_VIEWS, N_PIX, world, rank)
    torch.save(res, out % rank)
    dist.destroy_process_group()


def test_two_rank_gather_equals_single_rank(tmp_path):
    from ngp_pl_b200.metrics import gather_metrics
    out = str(tmp_path / "metrics_r%d.pt")
    mp.spawn(_worker, args=(2, _free_port(), out), nprocs=2, join=True)
    single = gather_metrics(_rows(), N_VIEWS, N_PIX)
    rows = _rows().tolist()
    want_psnr = [-10 * math.log10(r[0] / (3 * N_PIX)) if r[0] > 0 else math.inf for r in rows]
    assert single["psnr_per_view"] == want_psnr
    assert single["ssim_per_view"] == [r[1] for r in rows]
    assert single["psnr"] == math.inf  # a perfect view makes the mean infinite, as torch's mean does in the reference
    assert single["ssim"] == sum(r[1] for r in rows) / N_VIEWS
    assert single["total_samples"] == int(sum(r[2] for r in rows))
    for r in range(2):
        assert torch.load(out % r) == single  # every rank gets the whole result


def test_means_over_views():
    from ngp_pl_b200.metrics import gather_metrics
    rows = torch.tensor([[3.0 * 100 * 0.01, 0.5, 10], [3.0 * 100 * 1e-4, 0.7, 20]], dtype=torch.float64)
    res = gather_metrics(rows, 2, 100)
    assert res["psnr_per_view"] == [20.0, 40.0] and res["psnr"] == 30.0
    assert res["ssim"] == 0.6 and res["total_samples"] == 30
