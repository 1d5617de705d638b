"""`import fused_lamb_CUDA` for the reference's own FusedLAMBAMP (lamb_amp_opt/fused_lamb/fused_lamb.py:8): the reference's CUDA
extension compiled from its sources by oracle/build_ref.py into oracle/_ref/ (test / baseline infrastructure; never used by the
H100 product path)."""
import os
import sys

_ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
if _ROOT not in sys.path:
    sys.path.insert(0, _ROOT)
from oracle import build_ref as _b  # noqa: E402

_ext = _b.load_module()
if _ext is None:
    raise ImportError("oracle/_ref/fused_lamb_CUDA*.so is missing: run `python oracle/build_ref.py` with DLE_REFERENCE_ROOT set to a reference checkout")
multi_tensor_l2norm = _ext.multi_tensor_l2norm
multi_tensor_lamb = _ext.multi_tensor_lamb
