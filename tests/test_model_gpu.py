"""GPU parity of the whole boundary: deeplearningexamples_b200.modeling.BertForPreTraining (bf16, sm_90a kernels)
vs (a) golden vectors produced by the reference's modeling.py (tests/golden/bert_small_golden.pt) and (b) the CPU
oracle run on the same weights, for forward logits/loss and every parameter gradient.

Tolerances (north_star): logits within 1e-2 relative (of the logit scale) in bf16; index gathers bit-exact."""
import os

import pytest
import torch

pytestmark = pytest.mark.gpu
bf = torch.bfloat16


def _build(cfg, sd, dense=True, dropout=0.0, dtype=bf):
    from deeplearningexamples_b200 import modeling
    c = modeling.BertConfig.from_dict({**cfg, "hidden_dropout_prob": dropout, "attention_probs_dropout_prob": dropout})
    m = modeling.BertForPreTraining(c, sequence_output_is_dense=dense)
    full = dict(sd)
    full["cls.predictions.decoder.weight"] = sd["bert.embeddings.word_embeddings.weight"]
    missing, unexpected = m.load_state_dict(full, strict=False)
    assert not missing and not unexpected, (missing, unexpected)
    return m.cuda().to(dtype).train()


def _criterion(scores, nsp, labels, nsl):
    flat = labels.view(-1)
    lf = torch.nn.CrossEntropyLoss(ignore_index=-1)
    return lf(scores.float().view(-1, scores.shape[-1]), flat[flat != -1]) + lf(nsp.float().view(-1, 2), nsl.view(-1))


def _rel(got, want):
    """max-norm relative error: max|got - want| / max|want|"""
    return ((got.float() - want.float()).abs().max() / want.float().abs().max().clamp_min(1e-12)).item()


def _rel_l2(got, want):
    """relative L2 error ||got - want|| / ||want||  (the 1e-2 bf16-logit bar of north_star is applied to this; a single bf16 ulp
    on one large logit already costs 0.4-0.8 % in the max-norm metric, which is therefore bounded more loosely)"""
    return ((got.float() - want.float()).norm() / want.float().norm().clamp_min(1e-12)).item()


@pytest.fixture(scope="module")
def small(golden_dir):
    from oracle import bert_oracle as O
    gold = torch.load(os.path.join(golden_dir, "bert_small_golden.pt"), weights_only=False)
    sd = O.bf16_representable_params(gold["cfg"], seed=gold["param_seed"])
    batch = O.synthetic_batch(2, 128, gold["cfg"]["vocab_size"], 10, seed=gold["batch_seed"], full_mask=False)
    return gold, sd, batch


def test_forward_backward_vs_reference_golden(small):
    gold, sd, batch = small
    m = _build(gold["cfg"], sd)
    b = {k: v.cuda() for k, v in batch.items()}
    scores, nsp = m(b["input_ids"], b["token_type_ids"], b["attention_mask"], b["labels"])
    assert scores.dtype == bf and scores.shape == gold["scores"].shape
    assert _rel_l2(scores.cpu(), gold["scores"]) < 1e-2 and _rel(scores.cpu(), gold["scores"]) < 2e-2
    assert _rel(nsp.cpu(), gold["nsp"]) < 2e-2
    loss = _criterion(scores, nsp, b["labels"], b["next_sentence_labels"])
    assert abs(loss.item() - gold["loss"].item()) < 2e-2 * gold["loss"].item()
    loss.backward()
    named = dict(m.named_parameters())
    for k, g in gold["grads"].items():
        got = named[k].grad.float().cpu()
        cos = torch.nn.functional.cosine_similarity(got.flatten(), g.float().flatten(), dim=0).item()
        assert cos > 0.995, (k, cos)
        assert _rel(got, g) < 5e-2, (k, _rel(got, g))
    for k, n in gold["grad_norms"].items():
        if k == "cls.predictions.decoder.weight" or k.endswith("key.bias"):
            continue          # tied weight; key.bias gradient is analytically zero (softmax shift invariance)
        assert named[k].grad is not None, k
        gn = named[k].grad.float().norm().item()
        assert abs(gn - n.item()) <= 5e-2 * n.item() + 1e-6, (k, gn, n.item())


def test_intermediate_activations_vs_reference_golden(small):
    gold, sd, batch = small
    m = _build(gold["cfg"], sd)
    b = {k: v.cuda() for k, v in batch.items()}
    acts = {}
    m.bert.encoder.layer[0].force_modular = True       # forward hooks on sub-modules need the module-by-module path
    m.bert.embeddings.register_forward_hook(lambda mod, i, o: acts.__setitem__("emb", o.detach()))
    m.bert.encoder.layer[0].attention.self.register_forward_hook(lambda mod, i, o: acts.__setitem__("ctx0", o.detach()))
    enc, _ = m.bert(b["input_ids"], b["token_type_ids"], b["attention_mask"])
    assert _rel(acts["emb"].cpu(), gold["embeddings"]) < 1e-2
    assert acts["ctx0"].shape == (128, 2, 256)                      # the layer-level API is (seq, bsz, hidden)
    assert _rel(acts["ctx0"].transpose(0, 1).cpu(), gold["layer0_ctx"]) < 2e-2
    assert _rel(enc[-1].cpu(), gold["seq_out"]) < 2e-2


def test_layer_api_seq_first_contiguous_equals_batch_first_view(small):
    """BertLayer.forward takes (seq, bsz, hidden) like the reference: a contiguous [S,B,H] tensor and the encoder's
    transposed view of a [B,S,H] buffer must give the same numbers."""
    gold, sd, batch = small
    m = _build(gold["cfg"], sd)
    layer = m.bert.encoder.layer[0]
    g = torch.Generator(device="cuda").manual_seed(3)
    x_bsh = torch.randn(2, 128, 256, generator=g, device="cuda").to(bf)
    mask = torch.zeros(2, 1, 1, 128, device="cuda")
    mask[1, :, :, 100:] = -10000.0
    y_view = layer(x_bsh.transpose(0, 1), mask)                       # batch-first memory, seq-first logical
    y_cont = layer(x_bsh.transpose(0, 1).contiguous(), mask)          # seq-first memory
    assert y_view.shape == y_cont.shape == (128, 2, 256)
    torch.testing.assert_close(y_view.float(), y_cont.float(), rtol=0, atol=0)


@pytest.mark.parametrize("B,S,full_mask", [(3, 256, True), (2, 384, False)])
def test_forward_vs_cpu_oracle_other_shapes(B, S, full_mask):
    from oracle import bert_oracle as O
    cfg = dict(hidden_size=512, num_hidden_layers=3, num_attention_heads=8, intermediate_size=2048, vocab_size=2048,
               max_position_embeddings=512, type_vocab_size=2, hidden_act="gelu", initializer_range=0.02)
    sd = O.bf16_representable_params(cfg, seed=33)
    batch = O.synthetic_batch(B, S, cfg["vocab_size"], 20, seed=9, full_mask=full_mask)
    with torch.no_grad():
        loss_ref, scores_ref, nsp_ref, seq_ref = O.forward_loss(sd, cfg, batch)
    m = _build(cfg, sd)
    b = {k: v.cuda() for k, v in batch.items()}
    with torch.no_grad():
        scores, nsp = m(b["input_ids"], b["token_type_ids"], b["attention_mask"], b["labels"])
    assert _rel_l2(scores.cpu(), scores_ref) < 1e-2 and _rel(scores.cpu(), scores_ref) < 3e-2
    loss = _criterion(scores, nsp, b["labels"], b["next_sentence_labels"])
    assert abs(loss.item() - loss_ref.item()) < 2e-2 * loss_ref.item()


def test_fp32_parameter_mode_matches_bf16_mode(small):
    """fp32 parameters (native-AMP style use): kernels run on cached bf16 copies; grads come back fp32."""
    gold, sd, batch = small
    m16, m32 = _build(gold["cfg"], sd), _build(gold["cfg"], sd, dtype=torch.float32)
    b = {k: v.cuda() for k, v in batch.items()}
    s16, n16 = m16(b["input_ids"], b["token_type_ids"], b["attention_mask"], b["labels"])
    s32, n32 = m32(b["input_ids"], b["token_type_ids"], b["attention_mask"], b["labels"])
    torch.testing.assert_close(s16.float(), s32.float(), rtol=0, atol=0)
    _criterion(s32, n32, b["labels"], b["next_sentence_labels"]).backward()
    p = dict(m32.named_parameters())["bert.encoder.layer.1.output.dense.weight"]
    assert p.grad.dtype == torch.float32
    g = gold["grad_norms"]["bert.encoder.layer.1.output.dense.weight"].item()
    assert abs(p.grad.norm().item() - g) < 5e-2 * g


def test_checkpoint_state_dict_round_trip(small, tmp_path):
    """state_dict keys are the reference's checkpoint names (399 for large incl. the tied decoder); save -> load is exact."""
    gold, sd, batch = small
    m = _build(gold["cfg"], sd)
    keys = set(m.state_dict().keys())
    assert "bert.encoder.layer.0.attention.self.query.weight" in keys and "cls.predictions.decoder.weight" in keys
    assert "bert.encoder.layer.1.intermediate.dense_act.bias" in keys and "bert.pooler.dense_act.weight" in keys
    path = tmp_path / "ckpt_1.pt"
    torch.save({"model": m.state_dict()}, path)
    m2 = _build(gold["cfg"], {k: torch.zeros_like(v) for k, v in sd.items()})
    m2.load_state_dict(torch.load(path)["model"], strict=False)
    for (k1, v1), (k2, v2) in zip(m.state_dict().items(), m2.state_dict().items()):
        assert k1 == k2 and torch.equal(v1, v2)
    att = m2.bert.encoder.layer[0].attention.self
    w, _ = att._packed()
    assert torch.equal(w[256:512], att.key.weight.data)


def test_dropout_training_step_runs_and_is_seed_deterministic(small):
    from deeplearningexamples_b200 import ops
    gold, sd, batch = small
    b = {k: v.cuda() for k, v in batch.items()}
    outs = []
    for _ in range(2):
        ops.manual_seed(1234)
        m = _build(gold["cfg"], sd, dropout=0.1)
        scores, nsp = m(b["input_ids"], b["token_type_ids"], b["attention_mask"], b["labels"])
        loss = _criterion(scores, nsp, b["labels"], b["next_sentence_labels"])
        loss.backward()
        outs.append((scores.detach().clone(), dict(m.named_parameters())["bert.encoder.layer.0.output.dense.weight"].grad.clone()))
    assert torch.equal(outs[0][0], outs[1][0])
    torch.testing.assert_close(outs[0][1].float(), outs[1][1].float(), rtol=1e-2, atol=1e-4)   # split-K atomics reorder fp32 adds
    m.eval()
    with torch.no_grad():
        s_eval, _ = m(b["input_ids"], b["token_type_ids"], b["attention_mask"], b["labels"])
    assert _rel_l2(s_eval.cpu(), gold["scores"]) < 1e-2 and not torch.equal(s_eval, outs[0][0])


def test_lamb_training_reduces_loss(small):
    """A few optimizer steps through the full boundary (model + FusedLAMBAMP + GradScaler + scheduler)."""
    from deeplearningexamples_b200.lamb import FusedLAMBAMP
    from deeplearningexamples_b200.schedulers import PolyWarmUpScheduler
    gold, sd, batch = small
    m = _build(gold["cfg"], sd)
    no_decay = ['bias', 'gamma', 'beta', 'LayerNorm']
    named = list(m.named_parameters())
    opt = FusedLAMBAMP([{'params': [p for n, p in named if not any(nd in n for nd in no_decay)], 'weight_decay': 0.01},
                        {'params': [p for n, p in named if any(nd in n for nd in no_decay)], 'weight_decay': 0.0}], lr=2e-3)
    sched = PolyWarmUpScheduler(opt, warmup=0.1, total_steps=40, base_lr=2e-3, device="cuda")
    scaler = torch.amp.GradScaler("cuda", init_scale=2.0 ** 10)
    opt.setup_fp32_params()
    b = {k: v.cuda() for k, v in batch.items()}
    losses = []
    for it in range(12):
        scores, nsp = m(b["input_ids"], b["token_type_ids"], b["attention_mask"], b["labels"])
        loss = _criterion(scores, nsp, b["labels"], b["next_sentence_labels"])
        losses.append(loss.item())
        scaler.scale(loss).backward()
        sched.step()
        scaler.step(opt)
        scaler.update()
        opt.zero_grad(set_to_none=True)
    assert opt.param_groups[0]['step'].item() == 12
    assert losses[-1] < losses[0] - 0.5, losses


def test_fused_layer_equals_modular_composition(small):
    """ops.BertLayerFn (default) vs the module-by-module composition: same forward bits, same gradients."""
    gold, sd, batch = small
    b = {k: v.cuda() for k, v in batch.items()}
    res = []
    for modular in (False, True):
        m = _build(gold["cfg"], sd)
        for layer in m.bert.encoder.layer:
            layer.force_modular = modular
        scores, nsp = m(b["input_ids"], b["token_type_ids"], b["attention_mask"], b["labels"])
        _criterion(scores, nsp, b["labels"], b["next_sentence_labels"]).backward()
        res.append((scores.detach(), {k: p.grad.detach().float() for k, p in m.named_parameters()}))
    assert torch.equal(res[0][0], res[1][0])
    for k in res[0][1]:
        if k.endswith("key.bias"):
            continue                                    # analytically zero gradient: both sides are rounding noise
        a, c = res[0][1][k], res[1][1][k]
        assert (a - c).abs().max().item() <= 2e-2 * c.abs().max().item() + 1e-6, k


def test_squad_head_forward_backward_vs_oracle():
    """BASELINE configs[3] shape (seq 384, QA head): BertForQuestionAnswering over the same encoder kernels vs the CPU oracle,
    and one FusedAdam + clip step (the SQuAD optimizer)."""
    from deeplearningexamples_b200 import modeling
    from deeplearningexamples_b200.adam import FusedAdam
    from oracle import bert_oracle as O
    cfg = dict(hidden_size=256, num_hidden_layers=2, num_attention_heads=4, intermediate_size=1024, vocab_size=1024,
               max_position_embeddings=512, type_vocab_size=2, hidden_act="gelu", initializer_range=0.02,
               hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
    sd = O.bf16_representable_params(cfg, seed=5)
    g = torch.Generator().manual_seed(6)
    qa_w = (torch.randn(2, 256, generator=g) * 0.05).to(bf).float()
    qa_b = torch.zeros(2)
    B, S = 2, 384
    batch = O.synthetic_batch(B, S, cfg["vocab_size"], 1, seed=8, full_mask=False)
    start, end = torch.randint(0, S, (B,), generator=g), torch.randint(0, S, (B,), generator=g)
    with torch.no_grad():
        seq, _ = O.bert_model(sd, cfg, batch["input_ids"], batch["token_type_ids"], batch["attention_mask"])
        logits_ref = torch.nn.functional.linear(seq, qa_w, qa_b)           # modeling.py:1366-1369
    m = modeling.BertForQuestionAnswering(modeling.BertConfig.from_dict(cfg))
    full = {k: v for k, v in sd.items() if k.startswith("bert.")}
    full["qa_outputs.weight"], full["qa_outputs.bias"] = qa_w, qa_b
    missing, unexpected = m.load_state_dict(full, strict=False)
    assert not missing and not unexpected, (missing, unexpected)
    m = m.cuda().to(bf).train()
    s_log, e_log = m(batch["input_ids"].cuda(), batch["token_type_ids"].cuda(), batch["attention_mask"].cuda())
    assert _rel_l2(s_log.cpu(), logits_ref[..., 0]) < 1e-2 and _rel_l2(e_log.cpu(), logits_ref[..., 1]) < 1e-2
    lf = torch.nn.CrossEntropyLoss()
    loss = (lf(s_log.float(), start.cuda()) + lf(e_log.float(), end.cuda())) / 2     # run_squad.py:1077-1080
    loss.backward()
    no_decay = ['bias', 'LayerNorm.bias', 'LayerNorm.weight']                          # run_squad.py:960-964
    named = list(m.named_parameters())
    opt = FusedAdam([{'params': [p for n, p in named if not any(nd in n for nd in no_decay)], 'weight_decay': 0.01},
                     {'params': [p for n, p in named if any(nd in n for nd in no_decay)], 'weight_decay': 0.0}], lr=3e-5,
                    bias_correction=False, max_grad_norm=1.0)
    opt.setup_fp32_params()
    before = named[10][1].detach().clone()
    opt.step()
    torch.cuda.synchronize()
    assert opt.param_groups[0]['step'].item() == 1 and opt._found_inf.item() == 0.0
    assert not torch.equal(before, named[10][1].detach())


def test_static_masked_count_is_equivalent_and_sync_free(small):
    """nonzero_static(batch*max_pred) gathers the same rows as torch.nonzero; surplus slots are ignored by the criterion."""
    from deeplearningexamples_b200.training import BertPretrainingCriterion
    gold, sd, batch = small
    b = {k: v.cuda() for k, v in batch.items()}
    m = _build(gold["cfg"], sd)
    crit = BertPretrainingCriterion(gold["cfg"]["vocab_size"], sequence_output_is_dense=True)
    s_dyn, n_dyn = m(b["input_ids"], b["token_type_ids"], b["attention_mask"], b["labels"])
    l_dyn = crit(s_dyn, n_dyn, b["labels"], b["next_sentence_labels"])
    m.cls.static_masked_count = 2 * 16                       # upper bound: 10 masked per sequence in this batch
    s_st, n_st = m(b["input_ids"], b["token_type_ids"], b["attention_mask"], b["labels"])
    assert s_st.shape[0] == 32 and torch.equal(s_st[:20], s_dyn)
    l_st = crit(s_st, n_st, b["labels"], b["next_sentence_labels"])
    assert abs(l_st.item() - l_dyn.item()) < 1e-3 * abs(l_dyn.item())
    l_st.backward()
    assert m.bert.embeddings.word_embeddings.weight.grad is not None


def test_bert_base_config0_shape_vs_reference_golden(golden_dir):
    """BASELINE.json configs[0] shape (BERT-base, B=4, S=128) on the GPU against the golden produced by the reference's own
    modeling.py in fp32.  Here the weights are NOT bf16-representable (N(0,0.02) fp32 init rounded to bf16 by the model cast), so
    this bounds the whole bf16 pipeline incl. weight rounding: loss within 1 %, logits within 2e-2 relative L2."""
    from oracle import bert_oracle as O
    gold = torch.load(os.path.join(golden_dir, "bert_base_golden.pt"), weights_only=False)
    cfg = gold["cfg"]
    sd = O.init_params(cfg, seed=gold["seed"])
    batch = O.synthetic_batch(4, 128, cfg["vocab_size"], 20, seed=gold["batch_seed"], full_mask=True)
    m = _build(cfg, sd)
    b = {k: v.cuda() for k, v in batch.items()}
    scores, nsp = m(b["input_ids"], b["token_type_ids"], b["attention_mask"], b["labels"])
    loss = _criterion(scores, nsp, b["labels"], b["next_sentence_labels"])
    assert abs(loss.item() - gold["loss"].item()) < 1e-2 * gold["loss"].item(), (loss.item(), gold["loss"].item())
    assert _rel_l2(scores[:8, :64].cpu(), gold["scores_slice"]) < 2e-2
    assert abs(scores.float().abs().mean().item() - gold["scores_absmean"].item()) < 2e-2 * gold["scores_absmean"].item()
    loss.backward()
    named = dict(m.named_parameters())
    for k, n in gold["grad_norms"].items():
        gn = named[k].grad.float().norm().item()
        assert abs(gn - n.item()) <= 6e-2 * n.item() + 1e-6, (k, gn, n.item())
