"""Padding-free inference route, the checks that need no GPU: argument validation of dle_attn_fwd_varlen, its header and ctypes
prototypes, and the refusal of the route outside inference."""
import ctypes
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    from deeplearningexamples_b200 import _lib as L
    if not os.path.exists(L.LIB_PATH):
        import __graft_entry__ as g
        g.build()
    return L.load()


def test_varlen_attention_rejects_invalid_arguments(lib):
    buf = ctypes.create_string_buffer(4096 + 16)
    p = ctypes.c_void_p((ctypes.addressof(buf) + 15) & ~15)            # 16-byte aligned; never dereferenced on these paths
    odd = ctypes.c_void_p(p.value + 2)
    good = (p, p, p, 2, 128, 16)
    assert lib.dle_attn_fwd_varlen(None, p, p, 2, 128, 16, None) == -22
    assert lib.dle_attn_fwd_varlen(p, None, p, 2, 128, 16, None) == -22
    assert lib.dle_attn_fwd_varlen(p, p, None, 2, 128, 16, None) == -22
    for B, S, A in [(0, 128, 16), (-1, 128, 16), (2, 128, 0), (2, 128, -3), (2, 0, 16), (2, -1, 16), (2, 513, 16), (2, 1024, 16)]:
        assert lib.dle_attn_fwd_varlen(p, p, p, B, S, A, None) == -22, (B, S, A)
    assert lib.dle_attn_fwd_varlen(odd, *good[1:], None) == -22                      # qkv not 16-byte aligned
    assert lib.dle_attn_fwd_varlen(p, p, odd, *good[3:], None) == -22                 # ctx not 16-byte aligned
    assert lib.dle_attn_fwd_varlen(p, ctypes.c_void_p(p.value + 1), p, *good[3:], None) == -22   # cu_seqlens not 4-byte aligned


def _strip_comments(txt):
    return re.sub(r"//[^\n]*", " ", re.sub(r"/\*.*?\*/", " ", txt, flags=re.S))


def test_varlen_prototypes_agree():
    from deeplearningexamples_b200 import _lib as L
    hdr = _strip_comments(open(os.path.join(ROOT, "include", "dle_b200.h")).read())
    m = re.search(r"int\s+dle_attn_fwd_varlen\s*\(([^;]*?)\)\s*;", hdr, flags=re.S)
    assert m, "dle_attn_fwd_varlen is not declared in include/dle_b200.h"
    params = [" ".join(a.split()) for a in m.group(1).split(",")]
    assert params == ["const void* qkv", "const int32_t* cu_seqlens", "void* ctx", "int32_t B", "int32_t max_seqlen", "int32_t A",
                      "void* stream"], params
    c = {"const void*": ctypes.c_void_p, "const int32_t*": ctypes.c_void_p, "void*": ctypes.c_void_p, "int32_t": ctypes.c_int32}
    want = [c[a.rsplit(" ", 1)[0]] for a in params]
    res, argtypes = L.SIGNATURES["dle_attn_fwd_varlen"]
    assert res is ctypes.c_int32 and argtypes == want


def _tiny_model(cls_name):
    from deeplearningexamples_b200 import modeling
    cfg = modeling.BertConfig(vocab_size_or_config_json_file=64, hidden_size=256, num_hidden_layers=1, num_attention_heads=4,
                              intermediate_size=1024, max_position_embeddings=64)
    return getattr(modeling, cls_name)(cfg)


@pytest.mark.parametrize("cls_name", ["BertModel", "BertForPreTraining", "BertForQuestionAnswering"])
def test_remove_padding_is_off_by_default_and_set_on_every_model_class(cls_name):
    m = _tiny_model(cls_name)
    bert = m if cls_name == "BertModel" else m.bert
    assert bert._remove_padding is False
    m.remove_padding(True)
    assert bert._remove_padding is True
    m.remove_padding(False)
    assert bert._remove_padding is False


def test_remove_padding_refuses_training_and_grad():
    from deeplearningexamples_b200 import _lib as L
    m = _tiny_model("BertModel")
    m.remove_padding(True)
    ids = torch.zeros(2, 16, dtype=torch.long)
    mask = torch.ones_like(ids)
    mask[1, 9:] = 0
    with pytest.raises(L.DleError, match="inference route"):
        m.train()(ids, torch.zeros_like(ids), mask)
    with pytest.raises(L.DleError, match="inference route"):
        m.eval()(ids, torch.zeros_like(ids), mask)                # eval mode, but grad enabled
