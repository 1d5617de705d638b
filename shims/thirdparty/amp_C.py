"""amp_C stand-in: reference fused_lamb.py:31-35 only stores amp_C.multi_tensor_l2norm / multi_tensor_lamb as attributes (its step()
calls fused_lamb_CUDA.* directly).  When the reference's own extension is importable the same callables are exposed."""
try:
    import fused_lamb_CUDA as _ext
    multi_tensor_l2norm = _ext.multi_tensor_l2norm
    multi_tensor_lamb = _ext.multi_tensor_lamb
except ImportError:                                        # H100 arm: the optimizer shim never touches these
    multi_tensor_l2norm = multi_tensor_lamb = None
