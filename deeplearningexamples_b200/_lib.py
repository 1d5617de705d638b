"""ctypes binding of libdle_b200.so (the C ABI declared in include/dle_b200.h).

There is no CPU fallback: if the shared library is missing or a call fails, an exception is
raised -- a silent eager/PyTorch path would void every parity and performance claim.
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# DLE_LIB_PATH: load another build of the SAME ABI (same-box A/B measurements of two kernel versions); default = the in-tree build
LIB_PATH = os.environ.get("DLE_LIB_PATH") or os.path.join(_HERE, "libdle_b200.so")

DLE_DTYPE_F32, DLE_DTYPE_BF16 = 0, 1
LAYOUT_K, LAYOUT_MN = 0, 1
(EPI_BIAS, EPI_BIAS_GELU, EPI_BIAS_DROPOUT_RESIDUAL, EPI_DGELU, EPI_ADD, EPI_ATOMIC_F32, EPI_F32,
 EPI_BIAS_TANH) = range(8)

_vp, _i32, _i64, _f32, _u32, _u64 = (ctypes.c_void_p, ctypes.c_int32, ctypes.c_int64, ctypes.c_float,
                                     ctypes.c_uint32, ctypes.c_uint64)


class GemmArgs(ctypes.Structure):
    _fields_ = [("A", _vp), ("B", _vp), ("out", _vp), ("out2", _vp), ("bias", _vp), ("aux", _vp),
                ("M", _i32), ("N", _i32), ("K", _i32), ("a_layout", _i32), ("b_layout", _i32),
                ("lda", _i64), ("ldb", _i64), ("ldo", _i64), ("ldo2", _i64), ("ld_aux", _i64),
                ("epilogue", _i32), ("splits", _i32), ("tile_n", _i32), ("alpha", _f32),
                ("dropout_p", _f32), ("dropout_stream", _u32), ("seed", _u64), ("seed_dev", _vp), ("colsum_out", _vp)]


class LambTensor(ctypes.Structure):
    _fields_ = [("grad", _vp), ("param", _vp), ("exp_avg", _vp), ("exp_avg_sq", _vp), ("model_param", _vp),
                ("numel", _i64), ("group", _i32), ("reserved", _i32)]


class LambGroup(ctypes.Structure):
    _fields_ = [("lr", _vp), ("step", _vp), ("beta1", _f32), ("beta2", _f32), ("eps", _f32),
                ("weight_decay", _f32), ("bias_correction", _i32), ("grad_averaging", _i32)]


# name -> (restype, argtypes): one entry per symbol declared in include/dle_b200.h
SIGNATURES = {
    "dle_version": (_i32, [ctypes.c_char_p, _i32]),
    "dle_gemm_bf16": (_i32, [ctypes.POINTER(GemmArgs), _vp]),
    "dle_attn_fwd": (_i32, [_vp, _vp, _vp, _vp, _i32, _i32, _i32, _i32, _f32, _u64, _vp, _u32, _vp]),
    "dle_attn_bwd": (_i32, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i32, _i32, _i32, _i32, _f32, _u64, _vp, _u32, _vp]),
    "dle_add_ln_fwd": (_i32, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _i32, _f32, _f32, _u64, _vp, _u32, _vp]),
    "dle_ln_bwd_partials": (_i32, [_i64]),
    "dle_ln_bwd_partials_h": (_i32, [_i64, _i32]),
    "dle_add_ln_bwd": (_i32, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _i32, _f32, _u64, _vp, _u32, _vp]),
    "dle_colsum_finalize": (_i32, [_vp, _i32, _i32, _vp, _i32, _i32, _vp]),
    "dle_colsum_finalize_batched": (_i32, [_vp, _i32, _i32, _i32, _vp, _i32, _i32, _vp]),
    "dle_colsum_partials": (_i32, [_i64]),
    "dle_colsum_bf16": (_i32, [_vp, _i64, _i32, _i64, _vp, _vp]),
    "dle_bias_gelu_fwd": (_i32, [_vp, _vp, _vp, _vp, _i64, _i32, _vp]),
    "dle_bias_gelu_bwd": (_i32, [_vp, _vp, _vp, _i64, _i32, _vp]),
    "dle_embed_ln_fwd": (_i32, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i32, _i32, _i32, _i32, _i32,
                                _i32, _f32, _f32, _u64, _vp, _u32, _vp, _vp]),
    "dle_embed_ln_bwd": (_i32, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i32, _i32, _i32, _f32,
                                _u64, _vp, _u32, _vp]),
    "dle_gather_rows": (_i32, [_vp, _vp, _vp, _i64, _i32, _i64, _vp, _vp]),
    "dle_scatter_rows": (_i32, [_vp, _vp, _vp, _i64, _i32, _i64, _vp]),
    "dle_advance_u64": (_i32, [_vp, _u64, _vp]),
    "dle_softmax_ce_fwd": (_i32, [_vp, _vp, _vp, _vp, _i64, _i32, _i64, _i64, _vp, _vp]),
    "dle_softmax_ce_bwd": (_i32, [_vp, _vp, _vp, _vp, _vp, _i64, _i32, _i64, _i64, _i64, _vp]),
    "dle_cast_f32_to_bf16": (_i32, [_vp, _vp, _i64, _vp]),
    "dle_cast_bf16_to_f32": (_i32, [_vp, _vp, _i64, _vp]),
    "dle_lamb_plan_create": (_i32, [ctypes.POINTER(LambTensor), _i32, ctypes.POINTER(LambGroup), _i32, _i32,
                                    ctypes.POINTER(_vp)]),
    "dle_lamb_plan_destroy": (_i32, [_vp]),
    "dle_lamb_plan_update": (_i32, [_vp, ctypes.POINTER(LambTensor), _i32, _vp]),
    "dle_lamb_step": (_i32, [_vp, _vp, _f32, _i32, _i32, _vp, _vp, _vp, _vp]),
    "dle_lamb_grad_norm": (_i32, [_vp, _vp, _vp, _vp]),
    "dle_adam_step": (_i32, [_vp, _vp, _f32, _f32, _i32, _vp, _vp, _vp]),
}

_ERRORS = {-22: "DLE_ERR_INVALID (bad shape/alignment/null pointer)", -5: "DLE_ERR_CUDA (launch/driver failure)",
           -38: "DLE_ERR_NOSYS (not compiled in)"}

_lib = None
# number of kernels of THIS library launched so far (bench.py reports it as gpu_launches)
launch_count = {"n": 0}


class DleError(RuntimeError):
    pass


def load():
    """Load the shared library (once) and set prototypes.  Raises if it is missing."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise DleError(
                f"{LIB_PATH} not found: build it with `python -m deeplearningexamples_b200.csrc.build` "
                "(there is no CPU/PyTorch fallback for the H100 hot path)")
        lib = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(lib, name)          # AttributeError if the .so lacks a declared symbol
            fn.restype, fn.argtypes = res, args
        _lib = lib
    return _lib


def check(rc, what):
    if rc != 0:
        raise DleError(f"{what} failed: {_ERRORS.get(rc, rc)}")
