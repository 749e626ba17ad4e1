"""Golden outputs of the network kernels on seeded inputs: the forward, the density lattice, the colour-MLP module and
the feature and weight gradients of the three backward kernels.

    python tests/golden/make_golden_network_core.py    rewrite tests/golden/network_core.npz (needs an H100)

What is stored is tests/test_network_core_gpu.py:network_core_outputs(): small runs as arrays, large runs as the SHA-256
of their output bytes. Regenerate only when what the network computes is meant to change.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

if __name__ == "__main__":
    from test_network_core_gpu import GOLDEN, network_core_outputs
    out = network_core_outputs()
    np.savez(GOLDEN, **out)
    print("%s: %d entries, %d bytes" % (GOLDEN, len(out), os.path.getsize(GOLDEN)))
