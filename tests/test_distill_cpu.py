"""General distillation, the parts that need no GPU: an fp32 restatement of the reference's losses (distillation/losses.py) and model
states (modeling.py) that the GPU tests compare against, the student's checkpoint keys, the layer mapping, the config refusals and the
argument checks of the new C entry points."""
import math
import types

import pytest
import torch
import torch.nn.functional as F

from deeplearningexamples_b200 import _lib as L

BACKBONE = {"distillation": True,
            "distillation_config": {"use_attention_scores": True, "use_hidden_states": True, "use_value_states": True,
                                    "use_embedding_states": False, "use_pred_states": False, "attention_loss": "kld",
                                    "hidden_state_loss": "cosine", "embedding_state_loss": "cosine", "value_state_loss": "kld",
                                    "student_teacher_layer_mapping": "last_layer"}}
SMALL = dict(hidden_size=128, num_hidden_layers=2, num_attention_heads=2, intermediate_size=512, vocab_size=512,
             max_position_embeddings=128, type_vocab_size=2, hidden_act="gelu", initializer_range=0.02,
             hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)


# ------------------------------------------------------------------------------------------------------------------------------
# fp32 restatement: materialised [B, A, S, S] tensors and torch autograd
# ------------------------------------------------------------------------------------------------------------------------------
def scores_from_qkv(qkv, mask, B, S, A, seq_first):
    """QK^T/sqrt(64) + mask [B, A, S, S] from a packed qkv [T, 3H] (modeling.py:349-361)."""
    H = A * 64
    x = qkv.float()
    x = x.view(S, B, 3 * H).transpose(0, 1) if seq_first else x.view(B, S, 3 * H)
    q = x[..., :H].reshape(B, S, A, 64).permute(0, 2, 1, 3)
    k = x[..., H:2 * H].reshape(B, S, A, 64).permute(0, 2, 1, 3)
    s = torch.matmul(q, k.transpose(-1, -2)) / 8.0
    return s if mask is None else s + mask.float().view(B, 1, 1, S)


def attention_kl(s_scores, t_scores):
    """losses.py:80-85 and :37-61 for one pair: where(x <= -100, 0, x), KLDivLoss(batchmean)(log_softmax(s), softmax(t)) / (A*S)."""
    s = torch.where(s_scores <= -1e2, torch.zeros_like(s_scores), s_scores)
    t = torch.where(t_scores <= -1e2, torch.zeros_like(t_scores), t_scores)
    A, S = s.shape[1], s.shape[-1]
    return F.kl_div(F.log_softmax(s, -1), F.softmax(t, -1), reduction="batchmean") / (A * S)


def value_kl(vs, vt, A_s, A_t, B):
    """losses.py:41-61: value states [S, B, A*d] -> per (b, h) V V^T / sqrt(d), then the KL above (no where rule)."""
    S = vs.shape[0]
    ds, dt = vs.shape[-1] // A_s, vt.shape[-1] // A_t
    sv = vs.float().reshape(S, B * A_s, ds).transpose(0, 1)
    tv = vt.float().reshape(S, B * A_t, dt).transpose(0, 1)
    p = (torch.bmm(sv, sv.transpose(1, 2)) / math.sqrt(ds)).view(B, A_s, S, S)
    t = (torch.bmm(tv, tv.transpose(1, 2)) / math.sqrt(dt)).view(B, A_t, S, S)
    return F.kl_div(F.log_softmax(p, -1), F.softmax(t, -1), reduction="batchmean") / (A_s * S)


def cosine_loss(pred, target, H):
    """losses.py:63-70: CosineEmbeddingLoss with target 1 over view(-1, H) rows."""
    return F.cosine_embedding_loss(pred.float().reshape(-1, H), target.float().reshape(-1, H), torch.ones(1, device=pred.device))


def model_states(sd, cfg, prefix, input_ids, token_type_ids, attention_mask):
    """fp32 BertModel forward that keeps the distillation states of the reference (modeling.py:298-300, 378-383, 458-461): embedding
    output [B, S, H], and per layer the scores [B, A, S, S], value states [S, B, H] and layer output [S, B, H]."""
    from oracle import bert_oracle as O
    A = cfg["num_attention_heads"]
    ext = O.extended_mask(attention_mask, torch.float32)
    emb = O.embeddings(sd, input_ids, token_type_ids, prefix=prefix + "embeddings.")
    h = emb.transpose(0, 1)
    S, B, H = h.shape
    out = {"embedding_states": emb, "attention_scores": [], "value_states": [], "hidden_states": []}
    for i in range(cfg["num_hidden_layers"]):
        p = f"{prefix}encoder.layer.{i}."
        a = p + "attention.self."
        q = F.linear(h, sd[a + "query.weight"], sd[a + "query.bias"]).view(S, B * A, 64).transpose(0, 1)
        k = F.linear(h, sd[a + "key.weight"], sd[a + "key.bias"]).view(S, B * A, 64).permute(1, 2, 0)
        v = F.linear(h, sd[a + "value.weight"], sd[a + "value.bias"]).view(S, B * A, 64).transpose(0, 1)
        scores = torch.bmm(q, k).view(B, A, S, S) / 8.0 + ext
        ctx = torch.bmm(F.softmax(scores, -1).view(B * A, S, S), v).transpose(0, 1).contiguous().view(S, B, H)
        x1 = O.layer_norm(F.linear(ctx, sd[p + "attention.output.dense.weight"], sd[p + "attention.output.dense.bias"]) + h,
                          sd[p + "attention.output.LayerNorm.weight"], sd[p + "attention.output.LayerNorm.bias"])
        inter = O.gelu_tanh(F.linear(x1, sd[p + "intermediate.dense_act.weight"], sd[p + "intermediate.dense_act.bias"]))
        h = O.layer_norm(F.linear(inter, sd[p + "output.dense.weight"], sd[p + "output.dense.bias"]) + x1,
                         sd[p + "output.LayerNorm.weight"], sd[p + "output.LayerNorm.bias"])
        out["attention_scores"].append(scores)
        out["value_states"].append(ctx)
        out["hidden_states"].append(h)
    return out


def distill_losses_fp32(s_states, t_states, s_cfg, t_cfg, dc, B, project=None):
    """general_distill.py:394-467: (att_loss, rep_loss, value_loss) from the two models' states; rep_loss includes the embedding
    term when dc["use_embedding_states"] is set."""
    n_s, n_t = len(s_states["hidden_states"]), len(t_states["hidden_states"])
    if dc["student_teacher_layer_mapping"] == "last_layer":
        pick = lambda s, t: ([s[-1]], [t[-1]])                                  # noqa: E731
    else:
        k = n_t // n_s
        pick = lambda s, t: (s, [t[i * k + k - 1] for i in range(n_s)])          # noqa: E731
    proj = (lambda xs: [F.linear(x, project[0], project[1]) for x in xs]) if project is not None else (lambda xs: xs)  # noqa: E731
    zero = torch.zeros(())
    att = rep = val = zero
    if dc["use_attention_scores"]:
        att = sum(attention_kl(s, t) for s, t in zip(*pick(s_states["attention_scores"], t_states["attention_scores"])))
    if dc["use_hidden_states"]:
        sr, tr = pick(s_states["hidden_states"], t_states["hidden_states"])
        rep = sum(cosine_loss(s, t, t_cfg["hidden_size"]) for s, t in zip(proj(sr), tr))
    if dc.get("use_embedding_states"):
        rep = rep + cosine_loss(proj([s_states["embedding_states"]])[0], t_states["embedding_states"], t_cfg["hidden_size"])
    if dc["use_value_states"]:
        val = sum(value_kl(s, t, s_cfg["num_attention_heads"], t_cfg["num_attention_heads"], B)
                  for s, t in zip(*pick(s_states["value_states"], t_states["value_states"])))
    return att, rep, val


# ------------------------------------------------------------------------------------------------------------------------------
# the restatement's own sanity: the where rule and the normalisation
# ------------------------------------------------------------------------------------------------------------------------------
def test_restated_attention_kl_matches_a_direct_sum():
    g = torch.Generator().manual_seed(0)
    s = torch.randn(2, 3, 8, 8, generator=g)
    t = torch.randn(2, 3, 8, 8, generator=g)
    s[0, 0, 0, 0] = -500.0                   # an unmasked score below -100: logit 0
    t[:, :, :, -1] = -10000.0                # a masked key: logit 0
    sw = torch.where(s <= -100, torch.zeros_like(s), s)
    tw = torch.where(t <= -100, torch.zeros_like(t), t)
    pt = F.softmax(tw, -1)
    direct = (pt * (F.log_softmax(tw, -1) - F.log_softmax(sw, -1))).sum() / (2 * 3 * 8)
    assert torch.allclose(attention_kl(s, t), direct, rtol=1e-6, atol=0)


def test_layer_mapping():
    from deeplearningexamples_b200 import distill as D
    assert D._layer_map(6, 12, "last_layer") is None
    assert D._layer_map(6, 12, "uniform") == [1, 3, 5, 7, 9, 11]
    assert D._layer_map(1, 2, "uniform") == [1]
    with pytest.raises(L.DleError, match="student_teacher_layer_mapping"):
        D._layer_map(5, 12, "uniform")


# ------------------------------------------------------------------------------------------------------------------------------
# model surface
# ------------------------------------------------------------------------------------------------------------------------------
def _write_config(tmp_path, cfg):
    import json
    (tmp_path / "config.json").write_text(json.dumps(cfg))
    (tmp_path / "distill.json").write_text(json.dumps(BACKBONE))
    return str(tmp_path), str(tmp_path / "distill.json")


def test_student_from_scratch_has_the_reference_keys(tmp_path):
    """BertForPreTraining.from_scratch(..., distill_config) has no cls heads and no pooler (modeling.py:639-653, 846-848, 940-958)."""
    from deeplearningexamples_b200 import modeling
    path, dc = _write_config(tmp_path, SMALL)
    student, config = modeling.BertForPreTraining.from_scratch(path, distill_config=dc)
    keys = set(student.state_dict())
    assert config.distillation and config.distillation_config["use_pooler"] is True
    assert not any(k.startswith("cls.") for k in keys) and not any(".pooler." in k for k in keys)
    assert "bert.encoder.layer.1.attention.self.query.weight" in keys and "bert.embeddings.word_embeddings.weight" in keys
    plain, _ = modeling.BertForPreTraining.from_scratch(path)
    assert keys == {k for k in plain.state_dict() if not k.startswith("cls.") and ".pooler." not in k}
    assert all(layer._distill_states() for layer in student.bert.encoder.layer)


def test_teacher_from_pretrained_with_distill_config(tmp_path):
    import json
    from deeplearningexamples_b200 import modeling
    path, dc = _write_config(tmp_path, SMALL)
    (tmp_path / "bert_config.json").write_text(json.dumps(SMALL))
    src = modeling.BertModel(modeling.BertConfig.from_dict(SMALL))
    torch.save({"bert." + k: v for k, v in src.state_dict().items()}, tmp_path / "pytorch_model.bin")
    teacher, config = modeling.BertModel.from_pretrained(path, distill_config=dc)
    teacher.make_teacher()
    assert teacher.teacher and config.distillation
    for k, v in teacher.state_dict().items():
        assert torch.equal(v, src.state_dict()[k]), k


def test_project_keys_and_init():
    from deeplearningexamples_b200 import modeling
    s_cfg = modeling.BertConfig.from_dict(dict(SMALL, hidden_size=64, num_attention_heads=1))
    t_cfg = modeling.BertConfig.from_dict(SMALL)
    torch.manual_seed(0)
    p = modeling.Project(s_cfg, t_cfg)
    assert list(p.state_dict()) == ["fit_dense.weight", "fit_dense.bias"]
    assert p.fit_dense.weight.shape == (128, 64) and torch.count_nonzero(p.fit_dense.bias) == 0
    assert abs(p.fit_dense.weight.std().item() - 0.02) < 0.003


def test_attention_scores_handle_shape_and_detach():
    from deeplearningexamples_b200 import modeling
    B, S, A = 2, 64, 2
    qkv = torch.randn(B * S, 3 * A * 64, requires_grad=True)
    mask = torch.zeros(B, S)
    mask[1, 40:] = -10000.0
    h = modeling.AttentionScores(qkv, mask, B, S, A, False)
    bsz, heads, s1, s2 = h.shape
    assert (bsz, heads, s1, s2) == (B, A, S, S)
    d = h.detach()
    assert not d.qkv.requires_grad and d.mask is mask
    assert torch.allclose(h.materialize(), scores_from_qkv(qkv, mask, B, S, A, False))


# ------------------------------------------------------------------------------------------------------------------------------
# refusals (no GPU needed: they are raised before any kernel runs)
# ------------------------------------------------------------------------------------------------------------------------------
def _cfgs(student=None, teacher=None, **dc):
    from deeplearningexamples_b200 import modeling
    s = modeling.BertConfig.from_dict(dict(SMALL, **(student or {})))
    t = modeling.BertConfig.from_dict(dict(SMALL, **(teacher or {})))
    d = {"distillation": True, "distillation_config": dict(BACKBONE["distillation_config"], **dc)}
    modeling._apply_distill_config(s, d, True)
    modeling._apply_distill_config(t, d, True)
    return s, t


@pytest.mark.parametrize("kw,match", [
    (dict(attention_loss="mse"), "attention_loss"),
    (dict(hidden_state_loss="mse"), "hidden_state_loss"),
    (dict(attention_loss="cosine"), "attention_loss"),
    (dict(value_state_loss="cosine"), "value_state_loss"),
])
def test_unbuilt_losses_are_refused(kw, match):
    from deeplearningexamples_b200 import distill as D
    s, t = _cfgs(**kw)
    with pytest.raises(L.DleError, match=match):
        D.TransformerLosses(s, t, "cpu", types.SimpleNamespace(train_batch_size=2))


def test_unbuilt_shapes_are_refused():
    from deeplearningexamples_b200 import distill as D
    s, t = _cfgs(student=dict(hidden_size=64, num_attention_heads=1))
    with pytest.raises(L.DleError, match="num_attention_heads"):
        D.check_distill_configs(s, t)
    s, t = _cfgs(student=dict(hidden_size=312, num_attention_heads=12), teacher=dict(hidden_size=768, num_attention_heads=12))
    with pytest.raises(L.DleError, match="head size"):
        D.check_distill_configs(s, t)


def test_distillation_layers_refuse_the_packed_routes():
    from deeplearningexamples_b200 import modeling
    s, _ = _cfgs()
    m = modeling.BertModel(s)
    with pytest.raises(L.DleError, match="no distillation"):
        m.encoder.layer[0].forward_packed(torch.zeros(4, 128), torch.zeros(2, dtype=torch.int32), 4)


def test_new_entry_points_validate_arguments(tmp_path):
    from deeplearningexamples_b200 import _lib
    import os
    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__ as g
        g.build()
    lib = _lib.load()
    assert lib.dle_relkl_partials(2, 128, 12) == 2 * 12 * 2
    assert lib.dle_relkl_partials(2, 100, 12) == -22
    assert lib.dle_relkl_fwd(None, None, None, None, 2304, 2304, None, None, 0.125, 0.125, 1, 2, 128, 12, 0, 1.0,
                             None, None, None, None, None) == -22
    assert lib.dle_relkl_bwd(None, None, None, None, 2304, 2304, None, None, 0.125, 0.125, 1, 2, 128, 12, 0, None, None, None, 1.0,
                             None, None, None, 2304, None) == -22
    assert lib.dle_cosine_rows_partials(130) == 3
    assert lib.dle_cosine_rows_fwd(None, 768, None, 768, 10, 768, None, None, None) == -22
    assert lib.dle_cosine_rows_bwd(None, 768, None, 768, 10, 768, None, None, 768, None) == -22
    assert lib.dle_add_rows_bf16(None, 8, None, 8, 4, 8, None, None) == -22


# ------------------------------------------------------------------------------------------------------------------------------
# the restatement against the reference's own code (tests/golden/make_distill_golden.py -> bert_distill_golden.pt)
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def distill_gold(golden_dir):
    import os
    return torch.load(os.path.join(golden_dir, "bert_distill_golden.pt"), weights_only=False)


def test_restatement_reproduces_the_reference_losses_and_gradients(distill_gold):
    """The fp32 restatement the GPU tests compare against reproduces the reference's modeling.py + hooks.py + losses.py + the layer
    mapping of general_distill.py: the where substitution, batchmean / (A*S), the value-relation view / transpose and the cosine rows."""
    from golden.make_distill_golden import B, CASES, STRIDE, TEACHER, distill_config, student_cfg, student_params, teacher_params
    b = distill_gold["batch"]
    assert [(c["n_student"], c["mapping"], c["use_embedding_states"]) for c in distill_gold["cases"]] == list(CASES)
    with torch.no_grad():
        t_states = model_states(teacher_params(), TEACHER, "bert.", b["input_ids"], b["token_type_ids"], b["attention_mask"])
    for case in distill_gold["cases"]:
        n = case["n_student"]
        s_cfg = student_cfg(n)
        sd = {k: v.clone().requires_grad_(True) for k, v in student_params(n).items()}
        s_states = model_states(sd, s_cfg, "bert.", b["input_ids"], b["token_type_ids"], b["attention_mask"])
        dc = distill_config(case["mapping"], case["use_embedding_states"])["distillation_config"]
        att, rep, val = distill_losses_fp32(s_states, t_states, s_cfg, TEACHER, dc, B)
        what = f"{n} layer(s), {case['mapping']}"
        for got, ref, name in ((att, case["att_loss"], "att"), (rep, case["rep_loss"], "rep"), (val, case["value_loss"], "value")):
            torch.testing.assert_close(got.detach(), ref, rtol=1e-5, atol=0, msg=lambda m, name=name: f"{what} {name}: {m}")
        (att + rep + val).backward()
        assert set(case["grad_keys"]) == set(sd), what
        torch.testing.assert_close(torch.stack([sd[k].grad.norm() for k in case["grad_keys"]]), case["grad_norms"], rtol=2e-4,
                                   atol=2e-6)
        strided = torch.cat([sd[k].grad.reshape(-1)[::STRIDE] for k in case["grad_keys"]])
        torch.testing.assert_close(strided, case["grads_strided"], rtol=2e-4, atol=2e-6)


def test_student_keys_equal_the_reference(distill_gold, tmp_path):
    """A distillation student built with from_scratch has the reference student's checkpoint keys, in order."""
    import json
    from deeplearningexamples_b200 import modeling
    from golden.make_distill_golden import distill_config, student_cfg
    for n, keys in distill_gold["state_dict_keys"].items():
        (tmp_path / "config.json").write_text(json.dumps(student_cfg(n)))
        student, _ = modeling.BertForPreTraining.from_scratch(str(tmp_path), distill_config=distill_config("last_layer", False))
        assert list(student.state_dict().keys()) == keys, n


def test_state_dict_key_mismatches_are_reported(caplog):
    import logging
    from deeplearningexamples_b200 import distill as D, modeling
    s, _ = _cfgs()
    m = modeling.BertModel(s)
    sd = dict(m.state_dict())
    sd.pop("embeddings.LayerNorm.bias")
    sd["pooler.dense_act.bias"] = torch.zeros(128)
    with caplog.at_level(logging.INFO, logger=D.__name__):
        D._load(m, sd, "teacher")
    text = caplog.text
    assert "teacher: weights not initialized" in text and "embeddings.LayerNorm.bias" in text
    assert "not used" in text and "pooler.dense_act.bias" in text
