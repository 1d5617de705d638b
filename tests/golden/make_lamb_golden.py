"""Write tests/golden/lamb_reference_kernel.npz: what the reference's own fused LAMB CUDA kernels (built into oracle/_ref by
oracle/build_ref.py from a checkout of the reference project) compute for the inputs of
tests/test_lamb_gpu.py::test_oracle_vs_reference_kernel.  Needs a GPU and the oracle/_ref build.

    python tests/golden/make_lamb_golden.py [OUT.npz]
"""
import importlib.util
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)


def main():
    spec = importlib.util.spec_from_file_location("test_lamb_gpu", os.path.join(ROOT, "tests", "test_lamb_gpu.py"))
    t = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(t)
    ext = t._ref_ext()
    if ext is None:
        raise SystemExit("oracle/_ref/fused_lamb_CUDA*.so is not built (python -m oracle.build_ref where the reference exists)")
    out = sys.argv[1] if len(sys.argv) > 1 else t.GOLDEN_LAMB
    np.savez_compressed(out, **t.reference_kernel_golden(ext))
    print("wrote", out)


if __name__ == "__main__":
    main()
