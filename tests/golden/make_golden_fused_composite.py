"""Golden outputs of the fused training kernel (k_train_composite_loss) on one seeded batch with a non-zero background.

    python tests/golden/make_golden_fused_composite.py    rewrite tests/golden/fused_composite.npz (needs an H100)

The batch and what is stored are those of tests/test_composite_core_gpu.py:fused_step_outputs(): per-ray rgb, opacity and
depth, per-sample dL/dsigma and dL/drgb in ray order, the loss scale, the per-ray sample counts, and a SHA-256 of the
network forward's outputs the kernel composited (the test checks it first, so a change to the network kernel is told
apart from one to compositing). Regenerate only when what the kernel computes is meant to change.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

if __name__ == "__main__":
    from test_composite_core_gpu import GOLDEN, fused_step_outputs
    out = fused_step_outputs()
    np.savez(GOLDEN, **out)
    print("%s: %d rays, %d samples" % (GOLDEN, out["rgb"].shape[0], out["dsigmas"].shape[0]))
