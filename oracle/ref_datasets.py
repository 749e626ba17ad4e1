"""The reference's dataset loaders, staged byte-identical into oracle/_ref/ngp_pl/datasets/ -- TEST INFRASTRUCTURE ONLY.

stage()          copies datasets/{base,nerf,colmap,colmap_utils,ray_utils,color_utils}.py from the reference tree (where it
                 exists; __graft_entry__.build() calls this next to build_ref.build()). Not its __init__.py, which
                 imports loaders outside this set: the staged directory is a namespace package
load(name)       imports the staged NeRFDataset / ColmapDataset with shims for the modules this machine lacks:
                 imageio.imread -> Pillow (the plugin imageio decodes PNG and JPEG with), kornia.create_meshgrid
                 (kornia.utils.grid.create_meshgrid with normalized_coordinates=False: torch.linspace(0, n-1, n) per axis,
                 stacked (x, y)) and tqdm (identity) when they are not installed

tests/golden/make_golden_datasets.py runs them on the fixtures; the goldens, not these modules, are what the tests read.
"""
import os
import shutil
import sys
import types

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get("NGP_REFERENCE_DIR", "/root/reference")
OUT = os.path.join(HERE, "_ref", "ngp_pl")
FILES = ["base.py", "nerf.py", "colmap.py", "colmap_utils.py", "ray_utils.py", "color_utils.py"]


def have_reference():
    return all(os.path.isfile(os.path.join(REF, "datasets", f)) for f in FILES)


def stage():
    d = os.path.join(OUT, "datasets")
    os.makedirs(d, exist_ok=True)
    for f in FILES:
        shutil.copyfile(os.path.join(REF, "datasets", f), os.path.join(d, f))
    return d


def _shims():
    import numpy as np
    import torch
    try:
        import imageio  # noqa: F401
    except ImportError:
        m = types.ModuleType("imageio")

        def imread(path):
            from PIL import Image
            with Image.open(path) as im:
                return np.array(im)
        m.imread = imread
        sys.modules["imageio"] = m
    try:
        import kornia  # noqa: F401
    except ImportError:
        m = types.ModuleType("kornia")

        def create_meshgrid(height, width, normalized_coordinates=True, device=None, dtype=torch.float32):
            assert not normalized_coordinates
            xs = torch.linspace(0, width - 1, width, device=device, dtype=dtype)
            ys = torch.linspace(0, height - 1, height, device=device, dtype=dtype)
            gx, gy = torch.meshgrid(xs, ys, indexing="xy")
            return torch.stack([gx, gy], -1)[None]
        m.create_meshgrid = create_meshgrid
        sys.modules["kornia"] = m
    try:
        import tqdm  # noqa: F401
    except ImportError:
        m = types.ModuleType("tqdm")
        m.tqdm = lambda it, *a, **k: it
        sys.modules["tqdm"] = m


def load(name):
    """the staged reference dataset class for 'nerf' or 'colmap'"""
    if not os.path.isdir(os.path.join(OUT, "datasets")):
        stage()
    _shims()
    if os.path.dirname(OUT) not in sys.path:
        sys.path.insert(0, os.path.dirname(OUT))
    if name == "nerf":
        from ngp_pl.datasets.nerf import NeRFDataset
        return NeRFDataset
    from ngp_pl.datasets.colmap import ColmapDataset
    return ColmapDataset
