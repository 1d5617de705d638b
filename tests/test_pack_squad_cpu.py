"""Packed SQuAD fine-tuning, the checks that need no GPU: the SQuAD packer's invariants and round trip, its position rules, a torch
restatement of dle_span_logits_unpack / dle_span_logits_pack_grad on a hand case (test_pack_squad_gpu.py compares the kernels with
it), the entry points' argument validation, and BertForQuestionAnswering's packing switch and refusals."""
import ctypes
import os

import numpy as np
import pytest
import torch

from deeplearningexamples_b200 import packing, squad
from test_pack_sequences_cpu import segment_table_ref

FILL = -10000.0


# ------------------------------------------------------------------------------------------------------------------------------
# restatement of the span-logit kernels (include/dle_b200.h)
# ------------------------------------------------------------------------------------------------------------------------------
def span_logits_ref(logits, cu, B, S, k, fill=FILL):
    """(start, end) [B*k, S] of logits [B*S, 2] (any dtype: the values are moved, fill rounded to the dtype)."""
    out = torch.full((2, B * k, S), fill, dtype=logits.dtype)
    cu = [int(c) for c in cu]
    for b in range(B):
        for j in range(k):
            seq = b * (k + 1) + j
            n = cu[seq + 1] - cu[seq]
            out[:, b * k + j, :n] = logits[cu[seq]:cu[seq] + n].t()
    return out[0], out[1]


def span_grad_ref(dstart, dend, cu, B, S, k):
    """dlogits [B*S, 2]: each sample token's two gradients, 0 at every tail token."""
    d = torch.zeros(B * S, 2, dtype=dstart.dtype)
    cu = [int(c) for c in cu]
    for b in range(B):
        for j in range(k):
            seq = b * (k + 1) + j
            n = cu[seq + 1] - cu[seq]
            d[cu[seq]:cu[seq] + n, 0] = dstart[b * k + j, :n]
            d[cu[seq]:cu[seq] + n, 1] = dend[b * k + j, :n]
    return d


def test_span_restatement_on_a_hand_case():
    B, S, k = 2, 6, 3
    mask = [[1, 1, 2, 3, 3, 0], [1, 1, 1, 1, 1, 1]]
    cu, _, _, bad = segment_table_ref(mask, k)
    assert bad == []
    logits = torch.arange(B * S * 2, dtype=torch.float32).view(B * S, 2)
    start, end = span_logits_ref(logits, cu, B, S, k)
    F = FILL
    assert start.tolist() == [[0, 2, F, F, F, F], [4, F, F, F, F, F], [6, 8, F, F, F, F],
                              [12, 14, 16, 18, 20, 22], [F] * 6, [F] * 6]
    assert end[0, :2].tolist() == [1, 3] and end[3].tolist() == [13, 15, 17, 19, 21, 23]
    d = span_grad_ref(start, end, cu, B, S, k)
    assert d[5].tolist() == [0, 0]                                     # the tail token
    assert torch.equal(d[:5], logits[:5]) and torch.equal(d[6:], logits[6:])


# ------------------------------------------------------------------------------------------------------------------------------
# SQuAD packer
# ------------------------------------------------------------------------------------------------------------------------------
def _source(n, B, S, seed):
    return [squad.synthetic_squad_features(B, S, 30522, seed=seed + i) for i in range(n)]


def _key(s):
    return (s.input_ids.tobytes(), s.segment_ids.tobytes(), s.start_position, s.end_position, s.feature_index)


def test_synthetic_features_put_answers_inside_each_feature():
    b = squad.synthetic_squad_features(64, 384, 30522, seed=3)
    lens = b["input_mask"].sum(1)
    assert int(lens.min()) >= 96 and int(lens.max()) <= 384 and bool((b["input_ids"][:, 0] == 101).all())
    assert bool((b["start_positions"] >= 0).all() and (b["start_positions"] <= b["end_positions"]).all())
    assert bool((b["end_positions"] < lens).all())
    assert bool((b["segment_ids"][b["input_mask"] == 0] == 0).all())


@pytest.mark.parametrize("B,S,k", [(16, 384, 3), (8, 128, 2), (32, 200, 8)])
def test_squad_packer_places_every_feature_once_within_the_row_bounds(B, S, k):
    src = _source(5, B, S, seed=10)
    want = sorted(_key(s) for i, b in enumerate(src) for s in packing.split_squad_samples(b, i * B))
    got = []
    for batch in packing.PackedLoader(src, B, S, k, squad=True):
        am, sp, ep, fi = batch["input_mask"], batch["start_positions"], batch["end_positions"], batch.feature_index
        assert am.shape == (B, S) and sp.shape == ep.shape == (B * k,) and fi.shape == (B * k,)
        assert all(batch[key].dtype == torch.int64 for key in packing.SQUAD_KEYS)
        _, _, _, bad = segment_table_ref(am.numpy(), k)
        assert bad == []
        for r in range(B):
            m = int(am[r].max())
            assert int((am[r] != 0).sum()) <= S and m <= k
            used = slice(r * k, r * k + m)
            empty = slice(r * k + m, (r + 1) * k)
            assert (fi[used] >= 0).all() and (fi[empty] == -1).all()
            assert bool((sp[empty] == S).all() and (ep[empty] == S).all())       # empty slots: ignore_index
            for j in range(1, m + 1):
                n = int((am[r] == j).sum())
                assert 0 <= int(sp[r * k + j - 1]) < n and 0 <= int(ep[r * k + j - 1]) < n
        samples = packing.unpack_squad(batch)
        assert len(samples) == batch.num_samples
        assert all(s.input_ids[0] == 101 for s in samples)
        got += [_key(s) for s in samples]
    assert sorted(got) == want


def test_unpack_squad_inverts_to_squad_batch():
    batch = _source(1, 12, 128, seed=4)[0]
    samples = packing.split_squad_samples(batch)
    rows, unplaced = packing.pack(samples, 12, 128, 4, 0)
    assert unplaced == []
    packed = packing.to_squad_batch(samples, rows, 12, 128, 4)
    back = packing.unpack_squad(packed)
    assert [_key(s) for s in back] == [_key(samples[i]) for r in rows for i in r]
    assert sorted(packed.feature_index[packed.feature_index >= 0].tolist()) == list(range(12))


def _one(n, start, end, S=64):
    s = packing.SquadSample(np.arange(n, dtype=np.int64), np.zeros(n, np.int64), start, end, 7)
    return packing.to_squad_batch([s], [[0]], 2, S, 2)


def test_positions_past_the_row_are_ignored_and_positions_in_the_padding_raise():
    b = _one(20, 3, 64 + 9)
    assert b["start_positions"].tolist() == [3, 64, 64, 64] and b["end_positions"].tolist() == [64, 64, 64, 64]
    assert b.feature_index.tolist() == [7, -1, -1, -1]
    assert _one(20, 64, 19)["start_positions"].tolist()[0] == 64
    for start, end in ((20, 5), (5, 63), (40, 41)):
        with pytest.raises(ValueError, match="padding"):
            _one(20, start, end)


def test_squad_split_refuses_packed_masks():
    batch = _source(1, 4, 64, seed=5)[0]
    with pytest.raises(ValueError, match="only 0 and 1"):
        packing.split_squad_samples(dict(batch, input_mask=batch["input_mask"] * 2))


def test_squad_fill_on_the_benchmark_distribution():
    """The bench's stream (tools/bench_squad_packed.py): B = 32, S = 384, k = 3."""
    B, S = 32, 384
    src = _source(8, B, S, seed=1)
    batches = list(packing.PackedLoader(src, B, S, 3, squad=True))
    unpacked = np.mean([packing.token_fill(b) for b in src])
    fill = np.mean([packing.token_fill(b) for b in batches[:-2]])
    print(f"token fill: packed {fill:.3f}, unpacked {unpacked:.3f}")
    assert fill > unpacked + 0.2


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


def test_span_entry_points_reject_invalid_arguments(lib):
    from deeplearningexamples_b200 import _lib as L
    buf = ctypes.create_string_buffer(4096 + 16)
    p = ctypes.c_void_p((ctypes.addressof(buf) + 15) & ~15)
    odd = ctypes.c_void_p(p.value + 1)
    two = ctypes.c_void_p(p.value + 2)
    bf, f32 = L.DLE_DTYPE_BF16, L.DLE_DTYPE_F32
    unpack = lambda lg, ld, cu, B, S, k, dt, s, e: lib.dle_span_logits_unpack(lg, ld, cu, B, S, k, dt, FILL, s, e, None)
    grad = lambda ds, de, cu, B, S, k, dt, d, ld: lib.dle_span_logits_pack_grad(ds, de, cu, B, S, k, dt, d, ld, None)
    for f in (unpack, grad):
        for i in range(4):                                        # every pointer
            ptrs = [p, p, p, p]
            ptrs[i] = None
            if f is unpack:
                assert f(ptrs[0], 2, ptrs[1], 4, 128, 3, bf, ptrs[2], ptrs[3]) == -22, i
            else:
                assert f(ptrs[0], ptrs[1], ptrs[2], 4, 128, 3, bf, ptrs[3], 2) == -22, i
        for B, S, k, dt, ld in [(0, 128, 3, bf, 2), (4, 0, 3, bf, 2), (4, 128, 0, bf, 2), (4, 128, -1, bf, 2), (16384, 128, 3, bf, 2),
                                (4, 128, 3, 2, 2), (4, 128, 3, -1, 2), (4, 128, 3, bf, 1)]:
            if f is unpack:
                assert f(p, ld, p, B, S, k, dt, p, p) == -22, (B, S, k, dt, ld)
            else:
                assert f(p, p, p, B, S, k, dt, p, ld) == -22, (B, S, k, dt, ld)
    assert unpack(odd, 2, p, 4, 128, 3, bf, p, p) == -22                   # bf16 needs 2-byte alignment
    assert unpack(two, 2, p, 4, 128, 3, f32, p, p) == -22                  # fp32 needs 4-byte alignment
    assert unpack(p, 2, two, 4, 128, 3, bf, p, p) == -22                   # cu_seqlens needs 4-byte alignment
    assert grad(p, p, p, 4, 128, 3, f32, two, 2) == -22


# ------------------------------------------------------------------------------------------------------------------------------
# model switch and refusals
# ------------------------------------------------------------------------------------------------------------------------------
def _qa(**cfg):
    from deeplearningexamples_b200 import modeling
    base = dict(vocab_size_or_config_json_file=64, hidden_size=256, num_hidden_layers=1, num_attention_heads=4, intermediate_size=1024,
                max_position_embeddings=64)
    base.update(cfg)
    return modeling.BertForQuestionAnswering(modeling.BertConfig(**base))


def _inputs(B=2, S=16):
    ids = torch.zeros(B, S, dtype=torch.long)
    mask = torch.ones_like(ids)
    mask[:, S // 2:] = 2
    return ids, torch.zeros_like(ids), mask


def test_question_answering_packing_switch():
    from deeplearningexamples_b200 import _lib as L
    m = _qa()
    assert m.bert._pack_per_row == 0 and not m._per_sample_logits
    with pytest.raises(L.DleError, match="per_sample_logits"):
        m.pack_sequences(3)
    assert m.bert._pack_per_row == 0
    m.pack_sequences(3, per_sample_logits=True)
    assert m.bert._pack_per_row == 3 and m._per_sample_logits
    m.pack_sequences(0)
    assert m.bert._pack_per_row == 0 and not m._per_sample_logits
    m.pack_sequences(None, per_sample_logits=True)
    assert m.bert._pack_per_row == 0 and not m._per_sample_logits
    with pytest.raises(L.DleError, match=">= 1"):
        m.pack_sequences(-1, per_sample_logits=True)
    # packing switched on below the QA model still refuses: the head would read rows, not samples
    m.bert.pack_sequences(2)
    with pytest.raises(L.DleError, match="QuestionAnswering"):
        m(*_inputs())


def _refused(m, inputs, match):
    from deeplearningexamples_b200 import _lib as L
    with pytest.raises(L.DleError, match=match):
        m(*inputs)


def test_question_answering_packed_route_refusals():
    m = _qa().train()
    m.pack_sequences(2, per_sample_logits=True)
    m.remove_padding(True, training=True)
    _refused(m, _inputs(), "remove_padding")
    m.remove_padding(False)
    m.checkpoint_activations(True)
    _refused(m, _inputs(), "checkpointing")
    m.checkpoint_activations(False)
    _refused(m, _inputs(S=128), "max_position_embeddings")
    _refused(m, _inputs(B=21846), "65535")
    m.bert.encoder.layer[0].force_modular = True
    _refused(m, _inputs(), "fused layer")
    m.bert.encoder.layer[0].force_modular = False
    _refused(m, _inputs(), "CUDA tensor")
    m2 = _qa(max_position_embeddings=1024)
    m2.pack_sequences(2, per_sample_logits=True)
    _refused(m2, _inputs(S=640), "S <= 512")
