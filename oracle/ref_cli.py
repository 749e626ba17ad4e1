"""The reference's command-line flags and checkpoint helpers, staged byte-identical into oracle/_ref/ngp_pl/ -- TEST
INFRASTRUCTURE ONLY.

stage()   copies opt.py and utils.py from the reference tree (where it exists; __graft_entry__.build() calls this next to
          build_ref.build() and ref_datasets.stage()). tests/test_train_cli_cpu.py parses the reference's own opt.py to
          check the flags of `python -m ngp_pl_b200.train`, and the CPU and GPU tests load the checkpoints it writes with
          the reference's own utils.load_ckpt / slim_ckpt. Both files import only argparse and torch.
"""
import os
import shutil

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get("NGP_REFERENCE_DIR", "/root/reference")
OUT = os.path.join(HERE, "_ref", "ngp_pl")
FILES = ["opt.py", "utils.py"]


def have_reference():
    return all(os.path.isfile(os.path.join(REF, f)) for f in FILES)


def stage():
    os.makedirs(OUT, exist_ok=True)
    for f in FILES:
        shutil.copyfile(os.path.join(REF, f), os.path.join(OUT, f))
    return OUT
