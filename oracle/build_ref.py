"""Build recipe for oracle/_ref: the reference's OWN fused LAMB CUDA extension, compiled from the sources where they
lie in a checkout of the reference project (REF_SRC; never copied), for sm_90a.  Output: oracle/_ref/fused_lamb_CUDA*.so (git-ignored).
TEST INFRASTRUCTURE ONLY: the GPU oracle for csrc/lamb.cu when it is present; tests/golden/lamb_reference_kernel.npz stores
what it computed so that the comparison also runs without it.

Sources: PyTorch/LanguageModeling/BERT/lamb_amp_opt/csrc/{frontend.cpp, multi_tensor_l2norm_kernel.cu, multi_tensor_lamb.cu}
Flags follow lamb_amp_opt/setup.py:10-27 (-O3 --use_fast_math -lineinfo, -DVERSION_GE_1_3 -DVERSION_GE_1_5).
"""
import glob
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
REF_SRC = "/root/reference/PyTorch/LanguageModeling/BERT/lamb_amp_opt/csrc"
if os.environ.get("DLE_REFERENCE_ROOT"):                 # another checkout of NVIDIA/DeepLearningExamples
    REF_SRC = os.path.join(os.environ["DLE_REFERENCE_ROOT"], "PyTorch/LanguageModeling/BERT/lamb_amp_opt/csrc")
# the reference's BERT example directory, read in place (never copied) by tools/run_reference_driver.py and the tests that run it
REF_BERT = os.path.dirname(os.path.dirname(REF_SRC))
OUT = os.path.join(HERE, "_ref")


def built_path():
    c = glob.glob(os.path.join(OUT, "fused_lamb_CUDA*.so"))
    return c[0] if c else None


def build_if_possible(force=False):
    if built_path() and not force:
        return built_path()
    if not os.path.isdir(REF_SRC):
        return None                      # no reference checkout: only a prebuilt file (if any) is used
    os.makedirs(OUT, exist_ok=True)
    os.environ.setdefault("TORCH_CUDA_ARCH_LIST", "9.0a")
    from torch.utils.cpp_extension import load
    srcs = [os.path.join(REF_SRC, f) for f in ("frontend.cpp", "multi_tensor_l2norm_kernel.cu", "multi_tensor_lamb.cu")]
    load(name="fused_lamb_CUDA", sources=srcs, build_directory=OUT, is_python_module=False, verbose=False,
         extra_cflags=["-O3", "-DVERSION_GE_1_1", "-DVERSION_GE_1_3", "-DVERSION_GE_1_5"],
         extra_cuda_cflags=["-O3", "--use_fast_math", "-lineinfo", "-DVERSION_GE_1_1", "-DVERSION_GE_1_3", "-DVERSION_GE_1_5",
                            "-gencode", "arch=compute_90a,code=sm_90a"])
    return built_path()


def load_module():
    """import the prebuilt reference extension (None if it is not there)."""
    p = built_path()
    if p is None:
        return None
    import importlib.util
    import torch  # noqa: F401  (the extension links against libtorch)
    spec = importlib.util.spec_from_file_location("fused_lamb_CUDA", p)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


if __name__ == "__main__":
    print(build_if_possible(force="--force" in sys.argv))
