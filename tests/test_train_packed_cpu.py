"""Padding-free training, the checks that need no GPU: argument validation of dle_attn_fwd_varlen_train and dle_attn_bwd_varlen,
their header and ctypes prototypes, the model switch and the route's refusals, and the driver's flag."""
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


def _aligned_ptr():
    buf = ctypes.create_string_buffer(4096 + 16)
    return buf, ctypes.c_void_p((ctypes.addressof(buf) + 15) & ~15)     # 16-byte aligned; never dereferenced on these paths


# (T, B, max_seqlen, A, drop_stride, dropout_p) that the entry points must reject
BAD_SIZES = [(0, 2, 128, 16, 128, 0.1), (-5, 2, 128, 16, 128, 0.1), (256, 0, 128, 16, 128, 0.1), (256, 65536, 128, 16, 128, 0.1),
             (256, 2, 0, 16, 128, 0.1), (256, 2, 513, 16, 512, 0.1), (256, 2, 128, 0, 128, 0.1), (256, 2, 128, 65536, 128, 0.1),
             (256, 2, 128, 16, 100, 0.1), (256, 2, 128, 16, 64, 0.1), (256, 2, 128, 16, 576, 0.1), (256, 2, 128, 16, 0, 0.1),
             (256, 2, 128, 16, 128, -0.1), (256, 2, 128, 16, 128, 1.0)]


def test_varlen_train_forward_rejects_invalid_arguments(lib):
    buf, p = _aligned_ptr()
    odd, odd4 = ctypes.c_void_p(p.value + 2), ctypes.c_void_p(p.value + 1)
    f = lib.dle_attn_fwd_varlen_train
    sizes = (256, 2, 128, 16, 128, 0.1, 7, None, 3, None)
    for i in range(4):                                                   # qkv, cu_seqlens, ctx, lse
        ptrs = [p, p, p, p]
        ptrs[i] = None
        assert f(*ptrs, *sizes) == -22, i
    for T, B, S, A, ds, dp in BAD_SIZES:
        assert f(p, p, p, p, T, B, S, A, ds, dp, 7, None, 3, None) == -22, (T, B, S, A, ds, dp)
    assert f(odd, p, p, p, *sizes) == -22                                # qkv not 16-byte aligned
    assert f(p, p, odd, p, *sizes) == -22                                # ctx not 16-byte aligned
    assert f(p, odd4, p, p, *sizes) == -22                               # cu_seqlens not 4-byte aligned
    assert f(p, p, p, odd4, *sizes) == -22                               # lse not 4-byte aligned


def test_varlen_backward_rejects_invalid_arguments(lib):
    buf, p = _aligned_ptr()
    odd, odd4 = ctypes.c_void_p(p.value + 2), ctypes.c_void_p(p.value + 1)
    f = lib.dle_attn_bwd_varlen
    tail = (256, 2, 128, 16, 128, 0.1, 7, None, 3, None)
    for i in range(7):                                                   # qkv, cu_seqlens, ctx, dctx, lse, dqkv, delta_ws
        ptrs = [p] * 8
        ptrs[i] = None
        assert f(*ptrs, *tail) == -22, i
    for T, B, S, A, ds, dp in BAD_SIZES:
        assert f(*([p] * 8), T, B, S, A, ds, dp, 7, None, 3, None) == -22, (T, B, S, A, ds, dp)
    for i in (0, 2, 3, 5):                                               # qkv, ctx, dctx, dqkv not 16-byte aligned
        ptrs = [p] * 8
        ptrs[i] = odd
        assert f(*ptrs, *tail) == -22, i
    for i in (1, 4, 6, 7):                                               # cu_seqlens, lse, delta_ws, dbias not 4-byte aligned
        ptrs = [p] * 8
        ptrs[i] = odd4
        assert f(*ptrs, *tail) == -22, i


def _strip_comments(txt):
    return re.sub(r"//[^\n]*", " ", re.sub(r"/\*.*?\*/", " ", txt, flags=re.S))


@pytest.mark.parametrize("name", ["dle_attn_fwd_varlen_train", "dle_attn_bwd_varlen"])
def test_varlen_train_prototypes_agree(name):
    from deeplearningexamples_b200 import _lib as L
    hdr = _strip_comments(open(os.path.join(ROOT, "include", "dle_b200.h")).read())
    m = re.search(r"int\s+%s\s*\(([^;]*?)\)\s*;" % name, hdr, flags=re.S)
    assert m, f"{name} is not declared in include/dle_b200.h"
    params = [" ".join(a.split()) for a in m.group(1).split(",")]
    c = {"const void*": ctypes.c_void_p, "void*": ctypes.c_void_p, "const int32_t*": ctypes.c_void_p, "const float*": ctypes.c_void_p,
         "float*": ctypes.c_void_p, "const uint64_t*": ctypes.c_void_p, "int32_t": ctypes.c_int32, "float": ctypes.c_float,
         "uint64_t": ctypes.c_uint64, "uint32_t": ctypes.c_uint32}
    want = [c[a.rsplit(" ", 1)[0]] for a in params]
    res, argtypes = L.SIGNATURES[name]
    assert res is ctypes.c_int32 and argtypes == want, params


def _tiny_model(cls_name):
    from deeplearningexamples_b200 import modeling
    cfg = modeling.BertConfig(vocab_size_or_config_json_file=64, hidden_size=256, num_hidden_layers=1, num_attention_heads=4,
                              intermediate_size=1024, max_position_embeddings=64)
    return getattr(modeling, cls_name)(cfg)


@pytest.mark.parametrize("cls_name", ["BertModel", "BertForPreTraining", "BertForQuestionAnswering"])
def test_remove_padding_training_flag_is_set_on_every_model_class(cls_name):
    m = _tiny_model(cls_name)
    bert = m if cls_name == "BertModel" else m.bert
    assert bert._remove_padding_training is False
    m.remove_padding(True, training=True)
    assert bert._remove_padding is True and bert._remove_padding_training is True
    m.remove_padding(True)
    assert bert._remove_padding is True and bert._remove_padding_training is False
    m.remove_padding(False, training=True)
    assert bert._remove_padding is False and bert._remove_padding_training is False


def _inputs():
    ids = torch.zeros(2, 16, dtype=torch.long)
    mask = torch.ones_like(ids)
    mask[1, 9:] = 0
    return ids, torch.zeros_like(ids), mask


def test_training_route_refuses_cuda_graph_capture(monkeypatch):
    from deeplearningexamples_b200 import _lib as L
    m = _tiny_model("BertModel").train()
    m.remove_padding(True, training=True)
    monkeypatch.setattr(torch.cuda, "is_current_stream_capturing", lambda: True)
    ids, tt, mask = _inputs()
    with pytest.raises(L.DleError, match="CUDA graph"):
        m(ids, tt, mask)


def test_training_route_refuses_activation_checkpointing():
    from deeplearningexamples_b200 import _lib as L
    m = _tiny_model("BertModel").train()
    m.remove_padding(True, training=True)
    m.checkpoint_activations(True)
    with pytest.raises(L.DleError, match="checkpointing"):
        m(*_inputs())


@pytest.mark.parametrize("bad", [2, -1])
def test_training_route_refuses_masks_other_than_0_1(bad):
    from deeplearningexamples_b200 import _lib as L
    m = _tiny_model("BertModel").train()
    m.remove_padding(True, training=True)
    ids, tt, mask = _inputs()
    mask[0, 3] = bad
    with pytest.raises(L.DleError, match="only 0 and 1"):
        m(ids, tt, mask)


@pytest.mark.parametrize("other", ["--cuda_graphs", "--checkpoint_activations"])
def test_driver_rejects_remove_padding_with(other):
    from deeplearningexamples_b200 import run_pretraining
    base = ["--config_file", "x.json", "--output_dir", "out", "--do_train"]
    assert run_pretraining.parse_arguments(base + ["--remove_padding"]).remove_padding is True
    assert run_pretraining.parse_arguments(base + [other]).remove_padding is False
    with pytest.raises(ValueError, match="--remove_padding"):
        run_pretraining.parse_arguments(base + ["--remove_padding", other])
