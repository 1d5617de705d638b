"""Write tests/golden/gemm_bitwise_digests.json: SHA-256 digests of what the GEMM computes for the cases of
tests/test_gemm_bitwise_gpu.py.  Needs a GPU; run it with the build whose results are to be pinned.

    python tests/golden/make_gemm_bitwise_golden.py [OUT.json]
"""
import importlib.util
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)


def main():
    spec = importlib.util.spec_from_file_location("test_gemm_bitwise_gpu", os.path.join(ROOT, "tests", "test_gemm_bitwise_gpu.py"))
    t = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(t)
    out = sys.argv[1] if len(sys.argv) > 1 else t.GOLDEN
    with open(out, "w") as f:
        json.dump(t.all_digests(), f, indent=1, sort_keys=True)
        f.write("\n")
    print("wrote", out)


if __name__ == "__main__":
    main()
