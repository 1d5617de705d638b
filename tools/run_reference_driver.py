#!/usr/bin/env python
"""Run an UNMODIFIED reference training script (read where it lies in the reference checkout, oracle/build_ref.py: REF_BERT) over either arm:

    python tools/run_reference_driver.py --arm ours      -- <run_pretraining.py flags>     # H100 kernels behind the reference names
    python tools/run_reference_driver.py --arm reference -- <run_pretraining.py flags>     # the reference's own modeling + CUDA LAMB
    python -m torch.distributed.run --nproc-per-node N ... tools/run_reference_driver.py --arm ours -- <flags>

--arm ours      : the script is copied ALONE into a scratch directory (so its sibling modules are not found next to it) and
                  `modeling`, `schedulers`, `lamb_amp_opt.fused_lamb`, `utils`, `file_utils` resolve to shims/ours/ (the H100 mirror).
--arm reference : the script runs in place beside the reference's own modeling.py / schedulers.py / lamb_amp_opt; the one
                  incompatibility with stock PyTorch is patched before it starts: modeling.gelu calls F.gelu(approximate=True), a
                  boolean only NVIDIA's container build accepts (modeling.py:121-122) -> approximate='tanh'.
Both arms get shims/thirdparty/ for the packages that are absent offline (lddl, dllogger, h5py, apex, amp_C, boto3).
"""
import argparse
import os
import runpy
import shutil
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle.build_ref import REF_BERT as REF  # noqa: E402
sys.dont_write_bytecode = True          # nothing is written into the reference checkout


def setup(arm, script="run_pretraining.py"):
    """Prepare sys.path / sys.modules for `arm`; returns the path of the script to execute."""
    src = os.path.join(REF, script)
    if not os.path.exists(src):
        raise SystemExit("%s is missing: no reference checkout (set DLE_REFERENCE_ROOT)" % src)
    third = os.path.join(ROOT, "shims", "thirdparty")
    if arm == "ours":
        scratch = tempfile.mkdtemp(prefix="dle_refscript_")
        path = os.path.join(scratch, script)
        shutil.copyfile(src, path)
        extra = [os.path.join(ROOT, "shims", "ours"), third, ROOT]
    elif arm == "reference":
        path = src
        extra = [REF, os.path.join(REF, "lamb_amp_opt"), os.path.join(ROOT, "shims", "reference"), third, ROOT]
    else:
        raise SystemExit("--arm must be ours or reference")
    for p in reversed(extra):
        if p in sys.path:
            sys.path.remove(p)
        sys.path.insert(0, p)
    if arm == "reference":
        import torch.nn.functional as F
        import modeling                     # the reference's own file (REF/modeling.py)
        modeling.gelu = lambda x: F.gelu(x, approximate="tanh")
        modeling.ACT2FN["gelu"] = modeling.gelu
    return path


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--arm", required=True, choices=["ours", "reference"])
    ap.add_argument("--script", default="run_pretraining.py")
    ap.add_argument("rest", nargs=argparse.REMAINDER)
    a = ap.parse_args()
    rest = a.rest[1:] if a.rest and a.rest[0] == "--" else a.rest
    path = setup(a.arm, a.script)
    sys.argv = [path] + rest
    runpy.run_path(path, run_name="__main__")


if __name__ == "__main__":
    main()
