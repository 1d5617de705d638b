"""Sequence packing, the checks that need no GPU: the host packer's invariants, determinism, round trip and fill; a pure-Python
restatement of dle_segment_table on hand cases (test_pack_sequences_gpu.py compares the kernel with it); the prototypes of the new and
changed entry points and their argument validation; the model switch and its refusals; the driver's flag."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

from deeplearningexamples_b200 import packing

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ------------------------------------------------------------------------------------------------------------------------------
# restatement of dle_segment_table (include/dle_b200.h)
# ------------------------------------------------------------------------------------------------------------------------------
def row_is_valid(row, k):
    prev = 0
    for s, v in enumerate(row):
        v = int(v)
        if v < 0 or v > k:
            return False
        if v != 0 and not (v == 1 if s == 0 else prev != 0 and v in (prev, prev + 1)):
            return False
        prev = v
    return True


def segment_table_ref(mask, k):
    """(cu_seqlens int32 [B*(k+1)+1], position_ids int64 [B, S], cls_index int64 [B*k], malformed rows) of a mask [B, S]."""
    mask = np.asarray(mask, dtype=np.int64)
    B, S = mask.shape
    cu = np.zeros(B * (k + 1) + 1, np.int64)
    pos = np.zeros((B, S), np.int64)
    cls = np.full(B * k, -1, np.int64)
    bad = []
    for b in range(B):
        row = mask[b]
        if not row_is_valid(row, k):
            bad.append(b)
            row = np.zeros(S, np.int64)                   # a malformed row is one tail segment
        starts = [b * S + int(np.argmax(row == j)) if (row == j).any() else None for j in range(1, k + 1)]
        n = int((row != 0).sum())
        for j in range(1, k + 1):
            cu[b * (k + 1) + j - 1] = starts[j - 1] if starts[j - 1] is not None else b * S + n
            if starts[j - 1] is not None:
                cls[b * k + j - 1] = starts[j - 1]
        cu[b * (k + 1) + k] = b * S + n
        for s in range(S):
            j = int(row[s])
            pos[b, s] = s - (starts[j - 1] - b * S if j else n)
    cu[B * (k + 1)] = B * S
    return cu.astype(np.int32), pos, cls, bad


def test_segment_table_restatement_on_hand_cases():
    k, S = 3, 8
    mask = [[1, 1, 1, 2, 2, 0, 0, 0],          # two samples and a tail
            [0] * 8,                            # no sample: all tail
            [1, 2, 2, 3, 3, 3, 3, 3],           # k samples, no tail, a length-1 sample
            [1] * 8,                            # one sample fills the row
            [1, 1, 3, 3, 0, 0, 0, 0],           # skipped number
            [1, 1, 0, 2, 0, 0, 0, 0],           # non-zero after 0
            [2, 2, 2, 0, 0, 0, 0, 0],           # does not start at 1
            [1, 2, 1, 0, 0, 0, 0, 0],           # decrease
            [1, 4, 0, 0, 0, 0, 0, 0]]           # value above k
    cu, pos, cls, bad = segment_table_ref(mask, k)
    assert bad == [4, 5, 6, 7, 8]
    assert cu[:8].tolist() == [0, 3, 5, 5, 8, 8, 8, 8]
    assert cu[8:16].tolist() == [16, 17, 19, 24, 24, 32, 32, 32]
    assert cu[-1] == 9 * 8
    for b in bad:                                         # one tail segment of length S
        assert cu[b * 4:b * 4 + 4].tolist() == [b * 8] * 4 and pos[b].tolist() == list(range(8))
        assert cls[b * 3:b * 3 + 3].tolist() == [-1] * 3
    assert pos[0].tolist() == [0, 1, 2, 0, 1, 0, 1, 2]
    assert pos[1].tolist() == list(range(8))
    assert pos[2].tolist() == [0, 0, 1, 0, 1, 2, 3, 4]
    assert cls[:12].tolist() == [0, 3, -1, -1, -1, -1, 16, 17, 19, 24, -1, -1]
    lens = np.diff(cu.astype(np.int64))
    assert (lens >= 0).all() and lens.sum() == 9 * 8      # every token in exactly one sequence


# ------------------------------------------------------------------------------------------------------------------------------
# host packer
# ------------------------------------------------------------------------------------------------------------------------------
def _source(n_batches, B, S, P, seed, round_to=1):
    return [packing.synthetic_varlen_batch(B, S, 30522, P, seed=seed + i, round_to=round_to) for i in range(n_batches)]


def _key(s):
    return (s.input_ids.tobytes(), s.token_type_ids.tobytes(), s.labels.tobytes(), s.next_sentence_label)


@pytest.mark.parametrize("B,S,k,P", [(16, 128, 3, 20), (8, 512, 2, 80), (32, 200, 8, 30)])
def test_packer_places_every_sample_once_within_the_row_bounds(B, S, k, P):
    src = _source(6, B, S, P, seed=10)
    want = sorted(_key(s) for b in src for s in packing.split_samples(b, P))
    got = []
    for batch in packing.PackedLoader(src, B, S, k, P):
        assert isinstance(batch, packing.PackedBatch)
        am, lab, nsl = batch["attention_mask"], batch["labels"], batch["next_sentence_labels"]
        assert am.shape == (B, S) and nsl.shape == (B, k) and all(batch[key].dtype == torch.int64 for key in packing.KEYS)
        cu, pos, cls, bad = segment_table_ref(am.numpy(), k)
        assert bad == []
        for r in range(B):
            m = int(am[r].max())
            assert int((am[r] != 0).sum()) <= S and m <= k and int((lab[r] != -1).sum()) <= P
            assert (nsl[r, :m] >= 0).all() and (nsl[r, m:] == -1).all()
            assert bool((lab[r][am[r] == 0] == -1).all())
        samples = packing.unpack(batch)
        assert len(samples) == batch.num_samples
        assert all(s.input_ids[0] == 101 for s in samples)                # each sample keeps its own [CLS]
        got += [_key(s) for s in samples]
    assert sorted(got) == want


def test_packer_is_deterministic_and_carries_leftovers():
    src = _source(5, 16, 128, 20, seed=3)
    a = list(packing.PackedLoader(src, 16, 128, 3, 20))
    b = list(packing.PackedLoader(src, 16, 128, 3, 20))
    assert len(a) == len(b) and all(torch.equal(x[key], y[key]) for x, y in zip(a, b) for key in packing.KEYS)
    assert [x.num_samples for x in a] == [y.num_samples for y in b]
    # more samples per batch than rows: some batches take samples of the next unpacked batch
    assert max(x.num_samples for x in a) > 16 and sum(x.num_samples for x in a) == 5 * 16


def test_unpack_inverts_to_batch():
    batch = _source(1, 12, 64, 10, seed=4)[0]
    samples = packing.split_samples(batch, 10)
    rows, unplaced = packing.pack(samples, 12, 64, 4, 10)
    assert unplaced == []
    packed = packing.to_batch(samples, rows, 12, 64, 4)
    back = packing.unpack(packed)
    assert [_key(s) for s in back] == [_key(samples[i]) for r in rows for i in r]


def test_fill_on_the_benchmark_distribution():
    """Lengths U{128..512} rounded up to 64 (tools/bench_train_packed.py), B = 128, S = 512, k = 3."""
    B, S = 128, 512
    src = _source(8, B, S, 80, seed=1, round_to=64)
    batches = list(packing.PackedLoader(src, B, S, 3, 80))
    unpacked_fill = np.mean([packing.token_fill(b) for b in src])
    full = batches[:-2]                                  # the last batches pack out the pool when the source ends
    fill = np.mean([packing.token_fill(b) for b in full])
    per_row = np.mean([b.num_samples / B for b in full])
    print(f"token fill: packed {fill:.3f} ({per_row:.2f} samples per row), unpacked {unpacked_fill:.3f}")
    assert fill >= 0.85 and fill > unpacked_fill + 0.1


def test_packer_refuses_samples_that_fit_no_row():
    batch = _source(1, 4, 64, 80, seed=5)[0]
    with pytest.raises(ValueError, match="max_predictions_per_seq"):
        packing.split_samples(batch, max_pred=1)
    with pytest.raises(ValueError, match="only 0 and 1"):
        packing.split_samples(dict(batch, attention_mask=batch["attention_mask"] * 2))


# ------------------------------------------------------------------------------------------------------------------------------
# C ABI
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def lib():
    from deeplearningexamples_b200 import _lib as L
    if not os.path.exists(L.LIB_PATH):
        import __graft_entry__ as g
        g.build()
    return L.load()


def _strip_comments(txt):
    return re.sub(r"//[^\n]*", " ", re.sub(r"/\*.*?\*/", " ", txt, flags=re.S))


@pytest.mark.parametrize("name", ["dle_segment_table", "dle_embed_ln_fwd", "dle_embed_ln_bwd"])
def test_prototypes_agree(name):
    from deeplearningexamples_b200 import _lib as L
    hdr = _strip_comments(open(os.path.join(ROOT, "include", "dle_b200.h")).read())
    m = re.search(r"int\s+%s\s*\(([^;]*?)\)\s*;" % name, hdr, flags=re.S)
    assert m, f"{name} is not declared in include/dle_b200.h"
    params = [" ".join(a.split()) for a in m.group(1).split(",")]
    want = [ctypes.c_void_p if "*" in a else {"int32_t": ctypes.c_int32, "float": ctypes.c_float, "uint64_t": ctypes.c_uint64,
                                              "uint32_t": ctypes.c_uint32}[a.rsplit(" ", 1)[0]] for a in params]
    res, argtypes = L.SIGNATURES[name]
    assert res is ctypes.c_int32 and argtypes == want, params
    assert params[-1] != "void* stream" or name == "dle_segment_table"
    if name != "dle_segment_table":
        assert params[-1] == "const int64_t* position_ids"


def test_segment_table_rejects_invalid_arguments(lib):
    buf = ctypes.create_string_buffer(4096 + 16)
    p = ctypes.c_void_p((ctypes.addressof(buf) + 15) & ~15)
    odd = ctypes.c_void_p(p.value + 4)
    f = lib.dle_segment_table
    ok = (4, 128, 3)
    for i in range(4):                                                   # mask, cu_seqlens, position_ids, cls_index
        ptrs = [p, p, p, p]
        ptrs[i] = None
        assert f(ptrs[0], *ok, *ptrs[1:], None, None) == -22, i
    for B, S, k in [(0, 128, 3), (4, 0, 3), (4, 128, 0), (4, 128, -1), (16384, 128, 3), (65535, 128, 1)]:
        assert f(p, B, S, k, p, p, p, None, None) == -22, (B, S, k)
    assert f(odd, *ok, p, p, p, None, None) == -22                       # mask not 8-byte aligned
    assert f(p, *ok, p, odd, p, None, None) == -22                       # position_ids not 8-byte aligned
    assert f(p, *ok, p, p, odd, None, None) == -22                       # cls_index not 8-byte aligned


# ------------------------------------------------------------------------------------------------------------------------------
# model switch and refusals
# ------------------------------------------------------------------------------------------------------------------------------
def _tiny_model(cls_name, **cfg):
    from deeplearningexamples_b200 import modeling
    base = dict(vocab_size_or_config_json_file=64, hidden_size=256, num_hidden_layers=1, num_attention_heads=4, intermediate_size=1024,
                max_position_embeddings=64)
    base.update(cfg)
    return getattr(modeling, cls_name)(modeling.BertConfig(**base))


def _inputs(B=2, S=16):
    ids = torch.zeros(B, S, dtype=torch.long)
    mask = torch.ones_like(ids)
    mask[:, S // 2:] = 2
    return ids, torch.zeros_like(ids), mask


@pytest.mark.parametrize("cls_name", ["BertModel", "BertForPreTraining"])
def test_pack_sequences_flag(cls_name):
    from deeplearningexamples_b200 import _lib as L
    m = _tiny_model(cls_name)
    bert = m if cls_name == "BertModel" else m.bert
    assert bert._pack_per_row == 0
    m.pack_sequences(3)
    assert bert._pack_per_row == 3
    m.pack_sequences(None)
    assert bert._pack_per_row == 0
    with pytest.raises(L.DleError, match=">= 1"):
        m.pack_sequences(-1)


def test_question_answering_refuses_packing():
    from deeplearningexamples_b200 import _lib as L
    m = _tiny_model("BertForQuestionAnswering")
    m.pack_sequences(0)
    with pytest.raises(L.DleError, match="QuestionAnswering"):
        m.pack_sequences(2)
    m.bert.pack_sequences(2)
    with pytest.raises(L.DleError, match="QuestionAnswering"):
        m(*_inputs())


def _refused(m, inputs, match):
    from deeplearningexamples_b200 import _lib as L
    with pytest.raises(L.DleError, match=match):
        m(*inputs)


def test_packed_route_refusals():
    m = _tiny_model("BertModel").train()
    m.pack_sequences(2)
    m.remove_padding(True, training=True)
    _refused(m, _inputs(), "remove_padding")
    m.remove_padding(False)
    m.checkpoint_activations(True)
    _refused(m, _inputs(), "checkpointing")
    m.checkpoint_activations(False)
    _refused(m, _inputs(S=128), "max_position_embeddings")
    _refused(m, _inputs(B=21846), "65535")
    m.encoder.layer[0].force_modular = True
    _refused(m, _inputs(), "fused layer")
    m.encoder.layer[0].force_modular = False
    m2 = _tiny_model("BertModel", hidden_size=512, num_attention_heads=4, max_position_embeddings=1024).train()     # head size 128
    m2.pack_sequences(2)
    _refused(m2, _inputs(), "fused layer")
    m3 = _tiny_model("BertModel", max_position_embeddings=1024)
    m3.pack_sequences(2)
    _refused(m3, _inputs(S=640), "S <= 512")


def test_packed_route_refuses_cpu_tensors():
    m = _tiny_model("BertForPreTraining").train()
    m.pack_sequences(2)
    ids, tt, mask = _inputs()
    _refused(m, (ids, tt, mask, torch.full_like(ids, -1)), "CUDA tensor")


# ------------------------------------------------------------------------------------------------------------------------------
# driver
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("other", ["--remove_padding", "--checkpoint_activations"])
def test_driver_rejects_pack_sequences_with(other):
    from deeplearningexamples_b200 import run_pretraining
    base = ["--config_file", "x.json", "--output_dir", "out", "--do_train"]
    assert run_pretraining.parse_arguments(base).pack_sequences == 0
    assert run_pretraining.parse_arguments(base + ["--pack_sequences", "3", "--cuda_graphs"]).pack_sequences == 3
    assert run_pretraining.parse_arguments(base + [other]).pack_sequences == 0
    with pytest.raises(ValueError, match="--pack_sequences"):
        run_pretraining.parse_arguments(base + ["--pack_sequences", "3", other])
    with pytest.raises(ValueError, match="--pack_sequences"):
        run_pretraining.parse_arguments(base + ["--pack_sequences", "-1"])


def test_driver_synthetic_source_has_variable_length_samples():
    from deeplearningexamples_b200.run_pretraining import SyntheticPretrainLoader
    loader = SyntheticPretrainLoader(16, 128, 20, 1024, 4, base_seed=1, rank=0, variable_length=True)
    b = next(iter(loader))
    lens = b["attention_mask"].sum(1)
    assert int(lens.min()) >= 32 and int(lens.max()) <= 128 and len(set(lens.tolist())) > 4
    n_lab = (b["labels"] != -1).sum(1)
    assert bool((n_lab <= 20).all()) and bool(((n_lab - 0.15 * lens).abs() <= 1).all() | (n_lab == 20).all())
    assert bool((b["labels"][b["attention_mask"] == 0] == -1).all())
