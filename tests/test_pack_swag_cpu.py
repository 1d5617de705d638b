"""SWAG fine-tuning, the checks that need no GPU: the fp32 multiple-choice oracle against the reference's own BertForMultipleChoice
(tests/golden/make_mc_golden.py -> bert_mc_golden.pt), the mirror's checkpoint keys, the synthetic example layout, the SWAG packer's
groups, round trip and refusals, the loss over empty groups, the optimizer's parameter groups and the reference's schedule."""
import os

import numpy as np
import pytest
import torch

from deeplearningexamples_b200 import packing, swag
from test_pack_glue_cpu import sequence_classification

C = 4


# ------------------------------------------------------------------------------------------------------------------------------
# fp32 oracle of BertForMultipleChoice.forward
# ------------------------------------------------------------------------------------------------------------------------------
def multiple_choice(sd, cfg, input_ids, token_type_ids, attention_mask, num_choices=C):
    """BertForMultipleChoice.forward, modeling.py:1203-1212: the one-label sequence-classification oracle on the flattened
    [B*C, S] rows, then view(-1, num_choices)."""
    S = input_ids.shape[-1]
    logits = sequence_classification(sd, cfg, input_ids.reshape(-1, S), token_type_ids.reshape(-1, S), attention_mask.reshape(-1, S))
    return logits.view(-1, num_choices)


@pytest.fixture(scope="module")
def gold(golden_dir):
    return torch.load(os.path.join(golden_dir, "bert_mc_golden.pt"), weights_only=False)


def test_oracle_matches_reference_multiple_choice(gold):
    from golden.make_mc_golden import FULL_GRADS, STRIDE, TINY, mc_params
    b = gold["batch"]
    assert gold["num_choices"] == C and tuple(gold["logits"].shape) == (3, C)
    sd = {k: v.clone().requires_grad_(True) for k, v in mc_params(TINY).items()}
    logits = multiple_choice(sd, TINY, b["input_ids"], b["segment_ids"], b["input_mask"])
    loss = torch.nn.CrossEntropyLoss()(logits, b["label_ids"])
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
    from golden.make_mc_golden import TINY, mc_params
    cfg = dict(TINY, hidden_dropout_prob=0.1, attention_probs_dropout_prob=0.1)
    m = modeling.BertForMultipleChoice(modeling.BertConfig.from_dict(cfg), num_choices=C)
    assert list(m.state_dict().keys()) == gold["state_dict_keys"]
    assert m.num_choices == C and isinstance(m.dropout, torch.nn.Dropout) and m.dropout.p == 0.1
    assert tuple(m.classifier.weight.shape) == (1, cfg["hidden_size"]) and tuple(m.classifier.bias.shape) == (1,)
    m.load_state_dict(mc_params(TINY))
    import shims.ours.modeling as shim
    assert shim.BertForMultipleChoice is modeling.BertForMultipleChoice


def test_from_pretrained_takes_num_choices(tmp_path):
    from deeplearningexamples_b200 import modeling
    from golden.make_mc_golden import TINY, mc_params
    (tmp_path / "bert_config.json").write_text(modeling.BertConfig.from_dict(TINY).to_json_string())
    sd = {k: v for k, v in mc_params(TINY).items() if k.startswith("bert.")}
    torch.save(sd, tmp_path / "pytorch_model.bin")
    model, config = modeling.BertForMultipleChoice.from_pretrained(str(tmp_path), num_choices=C)
    assert isinstance(model, modeling.BertForMultipleChoice) and model.num_choices == C
    assert torch.equal(model.bert.embeddings.word_embeddings.weight, sd["bert.embeddings.word_embeddings.weight"])


# ------------------------------------------------------------------------------------------------------------------------------
# synthetic examples and the SWAG packer
# ------------------------------------------------------------------------------------------------------------------------------
def test_synthetic_features_share_a_context():
    b = swag.synthetic_swag_features(40, C, 128, 30522, seed=3)
    ids, am, seg = b["input_ids"], b["input_mask"], b["segment_ids"]
    assert ids.shape == am.shape == seg.shape == (40, C, 128) and b["label_ids"].shape == (40,)
    assert all(v.dtype == torch.int64 for v in b.values())
    assert set(b["label_ids"].tolist()) == set(range(C))
    contexts = []
    for n in range(40):
        ctx = None
        for c in range(C):
            L = int(am[n, c].sum())
            assert bool((am[n, c, :L] == 1).all()) and bool((am[n, c, L:] == 0).all())       # right-padded
            row = ids[n, c, :L]
            sep = torch.nonzero(row == 102).squeeze(-1).tolist()
            assert row[0] == 101 and len(sep) == 2 and sep[1] == L - 1 and sep[0] < L - 2
            assert bool((seg[n, c, :sep[0] + 1] == 0).all()) and bool((seg[n, c, sep[0] + 1:L] == 1).all())
            assert bool((ids[n, c, L:] == 0).all()) and bool((seg[n, c, L:] == 0).all())
            if ctx is None:
                ctx = row[1:sep[0]]
            assert torch.equal(row[1:sep[0]], ctx), (n, c)                                   # the same context in every choice
            assert 8 <= ctx.numel() <= 32 and 4 <= L - sep[0] - 2 <= 16
        contexts.append(ctx)
    assert len({c.numel() for c in contexts}) > 1
    with pytest.raises(ValueError, match="max_context"):
        swag.synthetic_swag_features(2, C, 64, 30522, max_context=50, max_ending=20)


def _source(n, N, S_choice, seed):
    return [swag.synthetic_swag_features(N, C, S_choice, 30522, seed=seed + i) for i in range(n)]


def _key(s):
    return (tuple(a.tobytes() for a in s.input_ids), tuple(a.tobytes() for a in s.segment_ids), s.label, s.example_index)


def _check_groups(batch, src, N, S, k):
    """Every example whole, its choices in order, at the C-aligned slots its group names; labels and example_index per group."""
    E = k // C
    am, lab, ei = batch["input_mask"].numpy(), batch["label_ids"].numpy(), batch.example_index
    B = am.shape[0]
    assert lab.shape == ei.shape == (B * E,)
    for r in range(B):
        nz = am[r][am[r] != 0]
        assert int((am[r] != 0).sum()) <= S and bool((am[r][len(nz):] == 0).all())               # the tail comes last
        assert bool((np.diff(nz) >= 0).all()) and (len(nz) == 0 or (nz.max() % C == 0 and nz.max() <= k))
        assert set(nz.tolist()) == set(range(1, int(nz.max(initial=0)) + 1))                       # whole examples, no gaps
        M = int(nz.max(initial=0)) // C
        used, empty = slice(r * E, r * E + M), slice(r * E + M, (r + 1) * E)
        assert (ei[used] >= 0).all() and (ei[empty] == -1).all() and (lab[empty] == -100).all()
        for m in range(M):
            e = int(ei[r * E + m])
            ex_ids, ex_am, ex_seg = (src[e // N][key][e % N] for key in ("input_ids", "input_mask", "segment_ids"))
            assert lab[r * E + m] == int(src[e // N]["label_ids"][e % N])
            for c in range(C):
                sel = am[r] == m * C + c + 1
                n = int(ex_am[c].sum())
                assert np.array_equal(batch["input_ids"][r].numpy()[sel], ex_ids[c, :n].numpy())
                assert np.array_equal(batch["segment_ids"][r].numpy()[sel], ex_seg[c, :n].numpy())


@pytest.mark.parametrize("B,S,k", [(32, 512, 16), (8, 256, 8), (6, 512, 4)])
def test_swag_packer_round_trip(B, S, k):
    N = 24
    src = _source(4, N, 128, seed=10)
    want = sorted(_key(s) for i, b in enumerate(src) for s in packing.split_swag_samples(b, i * N))
    got = []
    batches = list(packing.PackedLoader(src, B, S, k, swag=True, num_choices=C))
    for batch in batches:
        assert batch["input_mask"].shape == (B, S) and all(batch[key].dtype == torch.int64 for key in packing.SWAG_KEYS)
        _check_groups(batch, src, N, S, k)
        samples = packing.unpack_swag(batch, C)
        assert len(samples) == batch.num_samples == int((batch.example_index >= 0).sum())
        got += [_key(s) for s in samples]
    assert sorted(got) == want
    again = [_key(s) for batch in packing.PackedLoader(src, B, S, k, swag=True, num_choices=C) for s in packing.unpack_swag(batch, C)]
    assert again == got                                                                         # deterministic


def test_unpack_swag_inverts_to_swag_batch():
    batch = _source(1, 12, 128, seed=4)[0]
    samples = packing.split_swag_samples(batch, 100)
    assert [len(s) for s in samples] == [int(batch["input_mask"][n].sum()) for n in range(12)]
    rows, unplaced = packing.pack(samples, 6, 512, 16 // C, 0)
    assert unplaced == []
    packed = packing.to_swag_batch(samples, rows, 6, 512, 16, C)
    assert [_key(s) for s in packing.unpack_swag(packed, C)] == [_key(samples[i]) for r in rows for i in r]
    assert sorted(packed.example_index[packed.example_index >= 0].tolist()) == list(range(100, 112))
    group = {int(e): i for i, e in enumerate(packed.example_index) if e >= 0}
    for s in samples:
        assert int(packed["label_ids"][group[s.example_index]]) == s.label


def test_token_fill_on_both_layouts():
    src = _source(1, 16, 128, seed=6)[0]
    unpacked = float(src["input_mask"].sum()) / src["input_mask"].numel()
    assert packing.token_fill(src) == pytest.approx(unpacked)
    batch = next(iter(packing.PackedLoader([src], 4, 512, 16, swag=True, num_choices=C)))
    assert packing.token_fill(batch) == pytest.approx(float((batch["input_mask"] != 0).sum()) / (4 * 512))
    assert packing.token_fill(batch) > unpacked


def test_swag_packer_refusals():
    src = _source(1, 4, 64, seed=5)
    for kw in (dict(squad=True), dict(glue=True)):
        with pytest.raises(ValueError, match="one format"):
            packing.PackedLoader(src, 4, 256, 8, swag=True, **kw)
    for k in (6, 2, 3):
        with pytest.raises(ValueError, match="multiple of num_choices"):
            packing.PackedLoader(src, 4, 256, k, swag=True, num_choices=C)
    samples = packing.split_swag_samples(src[0])
    with pytest.raises(ValueError, match="multiple of num_choices"):
        packing.to_swag_batch(samples, [[0]], 4, 256, 6, C)
    with pytest.raises(ValueError, match="only 0 and 1"):
        packing.split_swag_samples(dict(src[0], input_mask=src[0]["input_mask"] * 2))
    partial = {k: v.clone() for k, v in src[0].items()}
    partial["input_mask"][1, 2] = 0
    with pytest.raises(ValueError, match="hold no token"):
        packing.split_swag_samples(partial)
    blank = {k: v.clone() for k, v in src[0].items()}
    blank["input_mask"][1] = 0
    assert [s.example_index for s in packing.split_swag_samples(blank)] == [0, 2, 3]                 # an all-padding example
    # an example longer than S: pack() and to_swag_batch() refuse it, as does the loader
    long = packing.SwagSample([np.arange(40, dtype=np.int64)] * C, [np.zeros(40, np.int64)] * C, 1, 0)
    with pytest.raises(ValueError, match="does not fit"):
        packing.pack([long], 4, 128, 16 // C, 0)
    with pytest.raises(ValueError, match="do not fit"):
        packing.to_swag_batch([long], [[0]], 4, 128, 16, C)
    with pytest.raises(ValueError, match="does not fit"):
        list(packing.PackedLoader(_source(1, 4, 128, seed=7), 4, 64, 16, swag=True, num_choices=C))
    # too many examples in a row, too many rows, the wrong number of choices
    with pytest.raises(ValueError, match="do not fit"):
        packing.to_swag_batch(samples, [[0, 1, 2]], 4, 512, 8, C)
    with pytest.raises(ValueError, match="rows do not fit"):
        packing.to_swag_batch(samples, [[0], [1], [2], [3]], 3, 512, 8, C)
    three = packing.SwagSample([np.arange(5, dtype=np.int64)] * 3, [np.zeros(5, np.int64)] * 3, 0, 0)
    with pytest.raises(ValueError, match="3 choices"):
        packing.to_swag_batch([three], [[0]], 1, 64, 4, C)


def test_loss_ignores_empty_groups_like_the_reference():
    """The reference's loss line on a packed batch: per-slot scores, view(-1, C), CrossEntropyLoss() with -100 in empty groups, is
    the mean over the real examples of their own C-way cross-entropy."""
    src = _source(1, 7, 64, seed=8)[0]
    samples = packing.split_swag_samples(src, 0)
    packed = packing.to_swag_batch(samples, [[0, 1, 2], [3], [], [4, 5, 6]], 5, 512, 12, C)
    g = torch.Generator().manual_seed(0)
    scores = torch.randn(7, C, generator=g)                                   # example e's C scores
    slots = torch.randn(5 * 12, generator=g)                                  # empty slots hold something finite
    for grp, e in enumerate(packed.example_index):
        if e >= 0:
            slots[grp * C:(grp + 1) * C] = scores[e]
    reshaped = slots.view(-1, C)
    assert reshaped.shape == (15, C) and int((packed["label_ids"] != -100).sum()) == 7
    got = torch.nn.CrossEntropyLoss()(reshaped, packed["label_ids"])
    want = torch.nn.CrossEntropyLoss()(scores, src["label_ids"])
    assert abs(got.item() - want.item()) < 1e-6
    terms = torch.nn.CrossEntropyLoss(reduction="none")(reshaped, packed["label_ids"])
    assert bool((terms[torch.from_numpy(packed.example_index < 0)] == 0).all())
    idx, pred = swag.swag_predictions(reshaped, packed)
    assert sorted(idx.tolist()) == list(range(7)) and all(pred[i] == int(scores[e].argmax()) for i, e in enumerate(idx))
    idx, pred = swag.swag_predictions(scores, dict(src))
    assert idx.tolist() == list(range(7)) and pred.tolist() == scores.argmax(-1).tolist()


# ------------------------------------------------------------------------------------------------------------------------------
# optimizer groups and the schedule (run_swag.py:406-431, 486-493)
# ------------------------------------------------------------------------------------------------------------------------------
class _RecordingAdam(torch.optim.SGD):
    """Stands in for FusedAdam on the CPU: keeps the groups and the keyword arguments it was built with."""

    def __init__(self, groups, lr, **kw):
        super().__init__(groups, lr=lr)
        self.kw = kw

    def setup_fp32_params(self):
        pass


TINY = dict(hidden_size=64, num_hidden_layers=2, num_attention_heads=4, intermediate_size=256, vocab_size=509,
            max_position_embeddings=64, type_vocab_size=2, hidden_act="gelu", initializer_range=0.02)


def test_optimizer_groups_leave_out_the_pooler(monkeypatch):
    monkeypatch.setattr(swag, "FusedAdam", _RecordingAdam)
    model, opt, sched = swag.prepare_swag_model_and_optimizer(TINY, torch.device("cpu"), total_steps=10, device_schedule=False)
    assert model.bert.embeddings.word_embeddings.weight.shape[0] == 512                       # vocabulary padded to a multiple of 8
    assert opt.kw == dict(bias_correction=False, max_grad_norm=1.0) and opt.defaults["lr"] == 5e-5
    by_id = {id(p): n for n, p in model.named_parameters()}
    decay, no_decay = ([by_id[id(p)] for p in g["params"]] for g in opt.param_groups)
    assert [g["weight_decay"] for g in opt.param_groups] == [0.01, 0.0]
    names = [n for n, _ in model.named_parameters()]
    assert sorted(decay + no_decay) == sorted(n for n in names if "pooler" not in n)
    assert not any("pooler" in n for n in decay + no_decay)
    assert all(n.endswith("bias") or "LayerNorm" in n for n in no_decay)
    assert not any(n.endswith("bias") or "LayerNorm" in n for n in decay)
    assert "classifier.weight" in decay and "classifier.bias" in no_decay
    for n, p in model.named_parameters():
        assert p.requires_grad == ("pooler" not in n), n


def test_host_schedule_is_the_reference_warmup_linear(monkeypatch):
    monkeypatch.setattr(swag, "FusedAdam", _RecordingAdam)
    total, warmup, base = 40, 0.1, 5e-5
    _, opt, sched = swag.prepare_swag_model_and_optimizer(TINY, torch.device("cpu"), total_steps=total, warmup_proportion=warmup,
                                                          learning_rate=base, device_schedule=False)
    for global_step in range(total + 3):
        sched.step()
        want = base * swag.warmup_linear(global_step / total, warmup)
        assert all(g["lr"] == pytest.approx(want, rel=1e-12, abs=1e-20) for g in opt.param_groups), (global_step, want)
        if global_step == 0:
            assert all(g["lr"] == 0.0 for g in opt.param_groups)
    # SQuAD and GLUE keep (step + 1) / total
    from deeplearningexamples_b200.schedulers import LinearWarmUpScheduler
    o = torch.optim.SGD([torch.nn.Parameter(torch.zeros(1))], lr=base)
    s = LinearWarmUpScheduler(o, warmup=warmup, total_steps=total)
    for n in range(total):
        s.step()
        assert o.param_groups[0]["lr"] == pytest.approx(base * swag.warmup_linear((n + 1) / total, warmup), rel=1e-12, abs=1e-20)


# ------------------------------------------------------------------------------------------------------------------------------
# refusals
# ------------------------------------------------------------------------------------------------------------------------------
def test_multiple_choice_refuses_cpu_tensors_and_misaligned_packing():
    from deeplearningexamples_b200 import _lib as L, modeling
    cfg = modeling.BertConfig(vocab_size_or_config_json_file=64, hidden_size=256, num_hidden_layers=1, num_attention_heads=4,
                              intermediate_size=1024, max_position_embeddings=64)
    m = modeling.BertForMultipleChoice(cfg, num_choices=C)
    ids = torch.zeros(2, C, 16, dtype=torch.long)
    with pytest.raises((L.DleError, RuntimeError)):
        m(ids, torch.zeros_like(ids), torch.ones_like(ids))
    for k in (1, 2, 6, 9, -4):
        with pytest.raises(L.DleError, match="multiple of num_choices"):
            m.pack_sequences(k)
        assert m.bert._pack_per_row == 0
    m.pack_sequences(8)
    assert m.bert._pack_per_row == 8
    with pytest.raises((L.DleError, RuntimeError)):
        m(ids[:, 0], torch.zeros_like(ids[:, 0]), torch.ones_like(ids[:, 0]))
    m.pack_sequences(0)
    assert m.bert._pack_per_row == 0
