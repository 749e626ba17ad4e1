"""Cost of the per-step training log (Trainer(log_rows=R): ngp_train_log_step at the end of every step, drain_log every 100
steps as `python -m ngp_pl_b200.train` does), one JSON line with the card's name and power limit:

  BASELINE config 2 (8192 rays, L=16, T=2^19, SynthLego bank of 100 views), the captured step with the log off and on,
  two trainers from the same seed, arms alternated window by window; ms per step of every window and the medians.

    python tools/train_log_cost.py [--steps 300] [--windows 7]
"""
import argparse
import json
import os
import statistics
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
from ngp_pl_b200 import synth  # noqa: E402
from ngp_pl_b200.models.networks import NGP  # noqa: E402
from ngp_pl_b200.trainer import Trainer  # noqa: E402
from eval_cost import card  # noqa: E402

DRAIN_EVERY = 100


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=300)
    ap.add_argument("--windows", type=int, default=7)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("train_log_cost.py measures on a CUDA device; none found")
    scene = synth.lego_scene(0)
    bank = synth.RayBank(scene, n_images=100, device="cuda")
    trs = {}
    for arm, rows in (("off", 0), ("on", 256)):
        torch.manual_seed(0)
        tr = Trainer(NGP(scene.scale).cuda(), n_rays=8192, log_rows=rows)
        tr.attach_bank(bank)
        tr.capture()
        for _ in range(300):
            tr.train_step()
            if rows and tr.host_step % DRAIN_EVERY == 0:
                tr.drain_log()
        trs[arm] = tr
    res = {k: [] for k in trs}
    logged = 0
    for _ in range(a.windows):
        for arm, tr in trs.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(a.steps):
                tr.train_step()
                if tr.log_ring is not None and tr.host_step % DRAIN_EVERY == 0:
                    logged += len(tr.drain_log())
            torch.cuda.synchronize()
            res[arm].append((time.perf_counter() - t0) * 1e3 / a.steps)
    logged += len(trs["on"].drain_log(wait=True))
    med = {k: statistics.median(v) for k, v in res.items()}
    print(json.dumps(dict(card=card(), steps_per_window=a.steps, step_ms_median=med, step_ms_windows=res,
                          log_cost_us_per_step=(med["on"] - med["off"]) * 1e3,
                          log_cost_fraction=(med["on"] - med["off"]) / med["off"], rows_logged=logged,
                          steps_on=trs["on"].host_step)))


if __name__ == "__main__":
    main()
