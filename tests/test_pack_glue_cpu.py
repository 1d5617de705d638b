"""GLUE fine-tuning, the checks that need no GPU: the fp32 sequence-classification oracle against the reference's own
BertForSequenceClassification (tests/golden/make_cls_golden.py -> bert_cls_golden.pt), the mirror's checkpoint keys, the GLUE packer's
round trip and refusals, and the argument validation of the head's entry points."""
import ctypes
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from deeplearningexamples_b200 import glue, packing
from oracle import bert_oracle as O


# ------------------------------------------------------------------------------------------------------------------------------
# fp32 oracle of the sequence-classification forward
# ------------------------------------------------------------------------------------------------------------------------------
def sequence_classification(sd, cfg, input_ids, token_type_ids, attention_mask, drop_keep=None, drop_scale=1.0):
    """BertForSequenceClassification.forward, modeling.py:1145-1155: classifier(dropout(pooled)) over oracle.bert_model's pooled
    output.  drop_keep [B, H] (1 = kept, kept values scaled by drop_scale) is the head's dropout mask; None omits it."""
    _, pooled = O.bert_model(sd, cfg, input_ids, token_type_ids, attention_mask)
    if drop_keep is not None:
        pooled = pooled * drop_keep.to(pooled.dtype) * drop_scale
    return F.linear(pooled, sd["classifier.weight"], sd["classifier.bias"])


@pytest.fixture(scope="module")
def gold(golden_dir):
    return torch.load(os.path.join(golden_dir, "bert_cls_golden.pt"), weights_only=False)


def test_oracle_matches_reference_classifier(gold):
    from golden.make_cls_golden import FULL_GRADS, STRIDE, TINY, cls_params
    b, L = gold["batch"], gold["num_labels"]
    sd = {k: v.clone().requires_grad_(True) for k, v in cls_params(TINY, L).items()}
    logits = sequence_classification(sd, TINY, b["input_ids"], b["segment_ids"], b["input_mask"])
    loss = torch.nn.CrossEntropyLoss()(logits.view(-1, L), b["label_ids"].view(-1))
    torch.testing.assert_close(logits, gold["logits"], rtol=1e-5, atol=1e-5)
    torch.testing.assert_close(loss, gold["loss"], rtol=1e-6, atol=1e-6)
    loss.backward()
    assert set(gold["grad_keys"]) == set(sd) and len(gold["grad_keys"]) == 41
    torch.testing.assert_close(torch.stack([sd[k].grad.norm() for k in gold["grad_keys"]]), gold["grad_norms"], rtol=2e-4, atol=2e-6)
    for k, g in gold["grads"].items():
        torch.testing.assert_close(sd[k].grad, g, rtol=2e-4, atol=2e-6, msg=lambda m, k=k: f"{k}: {m}")
    strided = torch.cat([sd[k].grad.reshape(-1)[::STRIDE] for k in gold["grad_keys"] if k not in FULL_GRADS])
    torch.testing.assert_close(strided, gold["grads_strided"], rtol=2e-4, atol=2e-6)


def test_mirror_state_dict_keys_equal_the_reference(gold):
    from deeplearningexamples_b200 import modeling
    from golden.make_cls_golden import TINY, cls_params
    cfg = dict(TINY, hidden_dropout_prob=0.1, attention_probs_dropout_prob=0.1)
    m = modeling.BertForSequenceClassification(modeling.BertConfig.from_dict(cfg), num_labels=gold["num_labels"])
    assert list(m.state_dict().keys()) == gold["state_dict_keys"]
    assert m.num_labels == 3 and isinstance(m.dropout, torch.nn.Dropout) and m.dropout.p == 0.1
    assert tuple(m.classifier.weight.shape) == (3, cfg["hidden_size"]) and not m.classifier.bias.any()
    m.load_state_dict(cls_params(TINY, 3))
    import shims.ours.modeling as shim
    assert shim.BertForSequenceClassification is modeling.BertForSequenceClassification


# ------------------------------------------------------------------------------------------------------------------------------
# GLUE packer
# ------------------------------------------------------------------------------------------------------------------------------
def _source(n, B, S, seed, num_labels=3):
    return [glue.synthetic_glue_features(B, S, 30522, num_labels, seed=seed + i) for i in range(n)]


def _key(s):
    return (s.input_ids.tobytes(), s.segment_ids.tobytes(), s.label, s.example_index)


def test_synthetic_features_are_sentence_pairs():
    b = glue.synthetic_glue_features(64, 128, 30522, 2, seed=3)
    lens = b["input_mask"].sum(1)
    assert int(lens.min()) >= 16 and int(lens.max()) <= 64
    assert bool((b["input_ids"][:, 0] == 101).all())
    for r in range(64):
        n = int(lens[r])
        sep = torch.nonzero(b["input_ids"][r, :n] == 102).squeeze(-1).tolist()
        assert len(sep) == 2 and sep[1] == n - 1 and 1 < sep[0] < n - 2
        assert b["segment_ids"][r, :sep[0] + 1].sum() == 0 and bool((b["segment_ids"][r, sep[0] + 1:n] == 1).all())
    assert bool((b["segment_ids"][b["input_mask"] == 0] == 0).all()) and set(b["label_ids"].tolist()) == {0, 1}


@pytest.mark.parametrize("B,S,k", [(32, 128, 4), (8, 128, 2), (16, 64, 6)])
def test_glue_packer_round_trip(B, S, k):
    src = _source(5, B, S, seed=10)
    want = sorted(_key(s) for i, b in enumerate(src) for s in packing.split_glue_samples(b, i * B))
    got = []
    for batch in packing.PackedLoader(src, B, S, k, glue=True):
        am, lab, ei = batch["input_mask"], batch["label_ids"], batch.example_index
        assert am.shape == (B, S) and lab.shape == (B * k,) and ei.shape == (B * k,)
        assert all(batch[key].dtype == torch.int64 for key in packing.GLUE_KEYS)
        for r in range(B):
            m = int(am[r].max())
            assert int((am[r] != 0).sum()) <= S and m <= k
            used, empty = slice(r * k, r * k + m), slice(r * k + m, (r + 1) * k)
            assert (ei[used] >= 0).all() and (ei[empty] == -1).all()
            assert bool((lab[empty] == -100).all()) and bool((lab[used] >= 0).all())
        samples = packing.unpack_glue(batch)
        assert len(samples) == batch.num_samples
        for s in samples:
            assert s.input_ids[0] == 101 and src[s.example_index // B]["label_ids"][s.example_index % B] == s.label
        got += [_key(s) for s in samples]
    assert sorted(got) == want
    again = [_key(s) for batch in packing.PackedLoader(src, B, S, k, glue=True) for s in packing.unpack_glue(batch)]
    assert again == got                                                                         # deterministic


def test_unpack_glue_inverts_to_glue_batch():
    batch = _source(1, 12, 128, seed=4)[0]
    samples = packing.split_glue_samples(batch, 100)
    rows, unplaced = packing.pack(samples, 12, 128, 4, 0)
    assert unplaced == []
    packed = packing.to_glue_batch(samples, rows, 12, 128, 4)
    assert [_key(s) for s in packing.unpack_glue(packed)] == [_key(samples[i]) for r in rows for i in r]
    assert sorted(packed.example_index[packed.example_index >= 0].tolist()) == list(range(100, 112))
    slot = {int(e): i for i, e in enumerate(packed.example_index) if e >= 0}
    for s in samples:
        assert int(packed["label_ids"][slot[s.example_index]]) == s.label


def test_glue_predictions_follow_the_slots():
    samples = [packing.GlueSample(np.arange(n, dtype=np.int64), np.zeros(n, np.int64), n % 3, 50 + n) for n in (5, 7, 9)]
    packed = packing.to_glue_batch(samples, [[0, 1], [2]], 3, 32, 2)
    logits = torch.zeros(6, 3)
    for slot, e in enumerate(packed.example_index):
        if e >= 0:
            logits[slot, int(e) % 3] = 1.0
    idx, pred = glue.glue_predictions(logits, packed)
    assert idx.tolist() == [55, 57, 59] and pred.tolist() == [55 % 3, 57 % 3, 59 % 3]
    idx, pred = glue.glue_predictions(logits[:4], {"input_ids": None})
    assert idx.tolist() == [0, 1, 2, 3]


def test_glue_packer_refusals():
    src = _source(1, 4, 64, seed=5)
    with pytest.raises(ValueError, match="one format"):
        packing.PackedLoader(src, 4, 64, 2, squad=True, glue=True)
    with pytest.raises(ValueError, match="only 0 and 1"):
        packing.split_glue_samples(dict(src[0], input_mask=src[0]["input_mask"] * 2))
    long = packing.GlueSample(np.arange(70, dtype=np.int64), np.zeros(70, np.int64), 1, 0)
    with pytest.raises(ValueError, match="does not fit"):
        packing.pack([long], 4, 64, 2, 0)
    with pytest.raises(ValueError, match="do not fit"):
        packing.to_glue_batch([long], [[0]], 4, 64, 2)
    with pytest.raises(ValueError):
        list(packing.PackedLoader([glue.synthetic_glue_features(4, 128, 30522, 3, seed=1, min_len=100, max_len=128)], 4, 64, 2,
                                  glue=True))


def test_loss_ignores_empty_slots_like_the_reference():
    logits = torch.randn(6, 3)
    labels = torch.tensor([0, 2, -100, 1, -100, -100])
    ref = torch.nn.CrossEntropyLoss()(logits[[0, 1, 3]], labels[[0, 1, 3]])
    torch.testing.assert_close(glue.glue_loss(logits.to(torch.bfloat16), labels),
                               torch.nn.CrossEntropyLoss()(logits.to(torch.bfloat16).float()[[0, 1, 3]], labels[[0, 1, 3]]))
    assert abs(glue.glue_loss(logits, labels).item() - ref.item()) < 1e-6


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


def test_head_entry_points_reject_invalid_arguments(lib):
    from deeplearningexamples_b200 import _lib as L
    buf = ctypes.create_string_buffer(4096 + 16)
    p = ctypes.c_void_p((ctypes.addressof(buf) + 15) & ~15)
    two = ctypes.c_void_p(p.value + 2)
    odd = ctypes.c_void_p(p.value + 1)
    bf, f32 = L.DLE_DTYPE_BF16, L.DLE_DTYPE_F32

    def fwd(x=p, ldx=64, w=p, b=p, R=4, H=64, L_=3, dt=bf, pd=0.1, out=p):
        return lib.dle_cls_head_fwd(x, ldx, w, b, R, H, L_, dt, pd, 1, None, 2, out, None)

    def bwd(d=p, x=p, ldx=64, w=p, R=4, H=64, L_=3, dt=bf, pd=0.1, dx=p, part=p, dw=p, db=p):
        return lib.dle_cls_head_bwd(d, x, ldx, w, R, H, L_, dt, pd, 1, None, 2, dx, part, dw, db, None)

    for f, ptr_names in ((fwd, ("x", "w", "b", "out")), (bwd, ("d", "x", "w", "dx", "part", "dw", "db"))):
        for name in ptr_names:
            assert f(**{name: None}) == -22, name
        for bad in (dict(L_=0), dict(L_=33), dict(L_=-1), dict(H=48), dict(H=0), dict(H=100), dict(R=0), dict(R=-3),
                    dict(dt=2), dict(dt=-1), dict(pd=1.0), dict(pd=-0.1), dict(ldx=32), dict(ldx=68), dict(x=two), dict(w=two)):
            assert f(**bad) == -22, (f.__name__, bad)
    assert fwd(b=odd) == -22 and fwd(dt=f32, out=two) == -22
    assert bwd(dt=f32, d=two) == -22 and bwd(dx=odd) == -22 and bwd(part=two) == -22
    assert lib.dle_cls_head_bwd_partials(0) == -22
    assert lib.dle_cls_head_bwd_partials(1) == 1 and lib.dle_cls_head_bwd_partials(128) == 4 and lib.dle_cls_head_bwd_partials(129) == 5


def test_sequence_classification_refuses_cpu_tensors():
    from deeplearningexamples_b200 import _lib as L, modeling
    cfg = modeling.BertConfig(vocab_size_or_config_json_file=64, hidden_size=256, num_hidden_layers=1, num_attention_heads=4,
                              intermediate_size=1024, max_position_embeddings=64)
    m = modeling.BertForSequenceClassification(cfg, num_labels=2)
    ids = torch.zeros(2, 16, dtype=torch.long)
    with pytest.raises((L.DleError, RuntimeError)):
        m(ids)
    m.pack_sequences(2)
    assert m.bert._pack_per_row == 2
    with pytest.raises((L.DleError, RuntimeError)):
        m(ids, torch.zeros_like(ids), torch.ones_like(ids))
