"""Stored outputs of oracle/grad64.py's mlp_backward on one seeded batch.

    python tests/golden/make_golden_grad64.py    rewrite tests/golden/grad64_mlp_backward.npz (CPU only)

tests/test_grad64_cpu.py:test_mlp_backward_unchanged recomputes them and compares. Regenerate only when what
mlp_backward computes is meant to change.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

if __name__ == "__main__":
    from test_grad64_cpu import GOLDEN_MLP, mlp_backward_outputs
    out = mlp_backward_outputs()
    np.savez_compressed(GOLDEN_MLP, **out)
    print("%s: %d arrays, %d bytes" % (GOLDEN_MLP, len(out), os.path.getsize(GOLDEN_MLP)))
