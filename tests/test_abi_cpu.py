"""C-ABI surface checks that need no GPU: include/dle_b200.h <-> exported symbols of libdle_b200.so <-> the ctypes table in
deeplearningexamples_b200/_lib.py, argument-validation returns (no compute is launched), and the "fail loudly" rule of the
product path (no CPU fallback)."""
import ctypes
import os
import re
import subprocess

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "dle_b200.h")


def _header_text():
    txt = open(HEADER).read()
    txt = re.sub(r"/\*.*?\*/", " ", txt, flags=re.S)
    return re.sub(r"//[^\n]*", " ", txt)


def _declared():
    """name -> number of parameters, for every function prototype in the header."""
    out = {}
    for m in re.finditer(r"\b(?:int|int32_t|const char\s*\*)\s+(dle_\w+)\s*\(([^;{]*?)\)\s*;", _header_text(), flags=re.S):
        args = m.group(2).strip()
        out[m.group(1)] = 0 if args in ("", "void") else args.count(",") + 1
    return out


@pytest.fixture(scope="module")
def lib():
    from deeplearningexamples_b200 import _lib as L
    if not os.path.exists(L.LIB_PATH):
        import __graft_entry__ as g
        g.build()
    return L.load()


def test_header_declares_the_reference_interfaces_it_replaces():
    raw = open(HEADER).read()
    assert 'extern "C"' in raw
    for cite in ("modeling.py", "fused_lamb.py", "multi_tensor_lamb.cu", "run_squad.py"):
        assert cite in raw, f"header must cite the reference interface in {cite}"
    assert "torch" not in _header_text().lower().replace("pytorch", ""), "no torch types in the C ABI"


def test_library_exports_exactly_the_declared_symbols(lib):
    from deeplearningexamples_b200 import _lib as L
    declared = _declared()
    assert len(declared) >= 25 and "dle_gemm_bf16" in declared and "dle_lamb_step" in declared
    nm = subprocess.run(["nm", "-D", "--defined-only", L.LIB_PATH], capture_output=True, text=True, check=True).stdout
    exported = {ln.split()[-1] for ln in nm.splitlines() if ln.split()[-1].startswith("dle_") and " T " in ln}
    assert exported == set(declared), f"header/library mismatch: only in header {set(declared) - exported}, only in .so {exported - set(declared)}"
    for name in declared:
        assert getattr(lib, name) is not None


def test_ctypes_table_matches_header_arity():
    from deeplearningexamples_b200 import _lib as L
    declared = _declared()
    assert set(L.SIGNATURES) == set(declared)
    for name, (_res, argtypes) in L.SIGNATURES.items():
        assert len(argtypes) == declared[name], f"{name}: ctypes has {len(argtypes)} args, header {declared[name]}"


def test_struct_layouts_match_header_field_order():
    from deeplearningexamples_b200 import _lib as L
    txt = _header_text()
    for cname, cls in (("dle_gemm_args", L.GemmArgs), ("dle_lamb_tensor", L.LambTensor), ("dle_lamb_group", L.LambGroup)):
        m = re.search(r"\{([^{}]*)\}\s*" + cname + r"\s*;", txt, flags=re.S)
        assert m, f"{cname} not found in header"
        fields = []
        for decl in (d.strip() for d in m.group(1).split(";")):
            if decl:                                        # "int32_t M, N, K" -> M, N, K ; "const void* A" -> A
                names = decl.split(",")
                fields.append(re.split(r"[\s\*]+", names[0].strip())[-1])
                fields += [n.strip().lstrip("*").strip() for n in names[1:]]
        assert fields == [f for f, _ in cls._fields_], f"{cname}: header {fields} vs ctypes {[f for f, _ in cls._fields_]}"
    assert ctypes.sizeof(L.LambTensor) == 56 and ctypes.sizeof(L.LambGroup) == 40   # 5 ptr + i64 + 2 i32 ; 2 ptr + 4 f32 + 2 i32


def test_version_and_argument_validation_without_a_gpu(lib):
    from deeplearningexamples_b200 import _lib as L
    buf = ctypes.create_string_buffer(64)
    assert lib.dle_version(buf, 64) >= 0
    assert b"sm_90a" in buf.value
    # preconditions are checked before any CUDA call: errno-style DLE_ERR_INVALID, never a crash
    assert lib.dle_gemm_bf16(None, None) == -22
    args = L.GemmArgs()                       # all-null pointers, zero sizes
    assert lib.dle_gemm_bf16(ctypes.byref(args), None) == -22
    assert lib.dle_attn_fwd(None, None, None, None, 1, 512, 16, 0, 0.0, 0, None, 0, None) == -22
    assert lib.dle_advance_u64(None, 1, None) == -22
    assert lib.dle_lamb_step(None, None, 1.0, 1, 0, None, None, None, None) == -22
    assert lib.dle_gather_rows(None, None, None, 0, 0, 0, None, None) == -22
    assert lib.dle_ln_bwd_partials(65536) > 0 and lib.dle_colsum_partials(65536) > 0      # pure host helpers


def test_product_path_fails_loudly_on_cpu_tensors():
    """No CPU fallback anywhere in the product path: CPU tensors (or a missing GPU) raise instead of silently computing."""
    from deeplearningexamples_b200 import kernels as k, _lib as L
    a = torch.zeros(128, 64, dtype=torch.bfloat16)
    with pytest.raises((L.DleError, RuntimeError)):
        k.gemm(a, a)
    from deeplearningexamples_b200 import modeling
    cfg = modeling.BertConfig(vocab_size_or_config_json_file=64, hidden_size=64, num_hidden_layers=1, num_attention_heads=1,
                              intermediate_size=256, max_position_embeddings=32)
    model = modeling.BertForPreTraining(cfg)
    ids = torch.zeros(2, 16, dtype=torch.long)
    with pytest.raises((L.DleError, RuntimeError)):
        model(ids, torch.zeros_like(ids), torch.ones_like(ids), torch.zeros_like(ids))


def test_product_code_never_imports_the_oracle():
    pkg = os.path.join(ROOT, "deeplearningexamples_b200")
    for dirpath, _dirs, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                src = open(os.path.join(dirpath, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle\b", src, flags=re.M), f"{f} imports oracle/"
                assert "liblamb_oracle" not in src and "bert_oracle" not in src, f"{f} references the oracle"
