"""Golden orbit-camera poses: the reference's OWN OrbitCamera (show_gui.py:19-51), driven by seeded input sequences.

    python tests/golden/make_golden_viewer.py    rewrite tests/golden/viewer_orbit.npz (needs the reference tree and scipy)

OrbitCamera is taken out of the reference's show_gui.py with `ast` (importing show_gui.py needs dearpygui, kornia and the
reference's CUDA extension) and executed with only numpy and scipy's Rotation in scope. Sequence s (s = 0 .. 39) starts
from OrbitCamera(K, (800, 800), r) with r drawn from [1, 4] and applies 1 to 30 calls, each drawn from:
  orbit(dx, dy)       dx, dy uniform in [-200, 200] (every 8th sequence: [-5000, 5000], many turns)
  scale(delta)        delta in {-1, +1} (the wheel) or uniform in [-3, 3]
  pan(dx, dy[, dz])   dx, dy uniform in [-3000, 3000]; dz too when the call's index is 2 mod 3
Stored per sequence: the radius, the calls (kind 0 orbit / 1 scale / 2 pan, then three arguments, unused ones 0, and
whether dz was passed) and `pose` after the last call. Regenerating gives byte-identical files (fixed seeds, np.savez
without compression and fixed key order).
"""
import ast
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get("NGP_REFERENCE_DIR", "/root/reference")
OUT = os.path.join(HERE, "viewer_orbit.npz")
N_SEQ = 40


def load_orbit_camera():
    src = open(os.path.join(REF, "show_gui.py")).read()
    cls = [n for n in ast.parse(src).body if isinstance(n, ast.ClassDef) and n.name == "OrbitCamera"][0]
    from scipy.spatial.transform import Rotation
    scope = {"np": np, "R": Rotation}
    exec(compile(ast.Module(body=[cls], type_ignores=[]), "show_gui.py", "exec"), scope)
    return scope["OrbitCamera"]


def sequences():
    """[(radius, calls (n, 5) float64: kind, a0, a1, a2, has_dz)] for every sequence, from seed 2024 + s"""
    out = []
    for s in range(N_SEQ):
        rng = np.random.RandomState(2024 + s)
        r = rng.uniform(1.0, 4.0)
        calls = []
        for _ in range(rng.randint(1, 31)):
            kind = rng.randint(3)
            if kind == 0:
                lim = 5000.0 if s % 8 == 7 else 200.0
                calls.append([0, rng.uniform(-lim, lim), rng.uniform(-lim, lim), 0, 0])
            elif kind == 1:
                d = float(rng.choice([-1, 1])) if rng.rand() < 0.5 else rng.uniform(-3, 3)
                calls.append([1, d, 0, 0, 0])
            else:
                has_dz = len(calls) % 3 == 2
                calls.append([2, rng.uniform(-3000, 3000), rng.uniform(-3000, 3000),
                              rng.uniform(-3000, 3000) if has_dz else 0.0, float(has_dz)])
        out.append((r, np.asarray(calls, np.float64)))
    return out


def apply(cam, calls):
    for kind, a0, a1, a2, has_dz in calls:
        if kind == 0:
            cam.orbit(a0, a1)
        elif kind == 1:
            cam.scale(a0)
        elif has_dz:
            cam.pan(a0, a1, a2)
        else:
            cam.pan(a0, a1)
    return cam.pose


def main():
    OrbitCamera = load_orbit_camera()
    K = np.float32([[1111.11, 0, 400], [0, 1111.11, 400], [0, 0, 1]])
    arrays = {}
    for s, (r, calls) in enumerate(sequences()):
        cam = OrbitCamera(K, (800, 800), r)
        arrays["radius_%02d" % s] = np.float64(r)
        arrays["calls_%02d" % s] = calls
        arrays["pose_%02d" % s] = apply(cam, calls)
    np.savez(OUT, **arrays)
    print("wrote %s (%d sequences)" % (OUT, N_SEQ))


if __name__ == "__main__":
    main()
