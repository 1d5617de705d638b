"""Generate the general-distillation golden vectors by running the UNMODIFIED reference modeling.py (BertModel as the teacher,
BertForPreTraining as the student, both built with a distillation config as from_scratch / from_pretrained build them,
modeling.py:644-648) with the reference's own distillation/hooks.py and distillation/losses.py, on CPU.  The layer mapping and the sum
of the three losses follow general_distill.py:394-467.  Imported as make_golden.py does, from $DLE_REFERENCE_ROOT.  Commit the output;
the tests themselves never need the reference.

    python tests/golden/make_distill_golden.py

Output
  bert_distill_golden.pt : a 2-layer teacher and students of 1 and 2 layers (H = 256, A = 4, d = 64, I = 1024, V = 512), B = 3,
                           S = 128 with ragged masks (one row of 17 tokens), dropout off.  Four cases: each student under the
                           "last_layer" and the uniform mapping; the 2-layer uniform case also turns on the embedding-state loss.
                           The parameters are regenerated from seeds by distill_params() (the tests call it too), so only outputs
                           are stored: the reference student's state_dict key list, the batch, and per case the attention, hidden
                           (+ embedding) and value losses, every student gradient's norm (in grad_keys order) and every STRIDE-th
                           element of each student gradient, concatenated in grad_keys order.
"""
import copy
import os
import sys
import types

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))

TEACHER = dict(hidden_size=256, num_hidden_layers=2, num_attention_heads=4, intermediate_size=1024, vocab_size=512,
               max_position_embeddings=128, type_vocab_size=2, hidden_act="gelu", initializer_range=0.02,
               hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
BACKBONE = {"distillation": True,
            "distillation_config": {"use_attention_scores": True, "use_hidden_states": True, "use_value_states": True,
                                    "use_embedding_states": False, "use_pred_states": False, "attention_loss": "kld",
                                    "hidden_state_loss": "cosine", "embedding_state_loss": "cosine", "value_state_loss": "kld",
                                    "student_teacher_layer_mapping": "last_layer"}}
# (student layers, mapping, use_embedding_states)
CASES = ((1, "last_layer", False), (1, "uniform", False), (2, "last_layer", False), (2, "uniform", True))
B, S = 3, 128
STRIDE = 997


def student_cfg(n_layers):
    return dict(TEACHER, num_hidden_layers=n_layers)


def distill_config(mapping, use_embedding_states):
    d = copy.deepcopy(BACKBONE)
    d["distillation_config"].update(student_teacher_layer_mapping=mapping, use_embedding_states=use_embedding_states)
    return d


def distill_params(cfg, seed):
    """Encoder + embedding parameters with the reference's BertForPreTraining names ("bert." prefix), from seeds: N(0, 0.1) weights,
    non-trivial LayerNorm affines and biases."""
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    from oracle import bert_oracle as O
    sd = {k: v for k, v in O.init_params(cfg, seed=seed, std=0.1).items() if k.startswith("bert.") and ".pooler." not in k}
    g = torch.Generator().manual_seed(seed + 1000)
    for k in sd:
        if "LayerNorm" in k or k.endswith("bias"):
            sd[k] = sd[k] + 0.1 * torch.randn(sd[k].shape, generator=g)
    return sd


def teacher_params():
    return distill_params(TEACHER, 51)


def student_params(n_layers):
    return distill_params(student_cfg(n_layers), 60 + n_layers)


def distill_batch():
    g = torch.Generator().manual_seed(29)
    ids = torch.randint(0, TEACHER["vocab_size"], (B, S), generator=g)
    ids[:, 0] = 101
    lens = torch.tensor([128, 70, 17])
    pos = torch.arange(S).unsqueeze(0)
    am = (pos < lens.unsqueeze(1)).long()
    seg = ((pos >= (lens // 2).unsqueeze(1)) & (am != 0)).long()
    return dict(input_ids=ids, token_type_ids=seg, attention_mask=am)


def _config(modeling, cfg, dc):
    config = modeling.BertConfig.from_dict(cfg)
    d = copy.deepcopy(dc)
    d["distillation_config"]["use_pooler"] = True                   # from_scratch / from_pretrained's default pooler=True
    config.__dict__.update(d)
    return config


def reference_losses(modeling, hooks, losses_mod, n_student, mapping, use_emb):
    """general_distill.py:380-467 with the reference's modules: (att_loss, rep_loss, value_loss, student model)."""
    dc = distill_config(mapping, use_emb)
    t_conf, s_conf = _config(modeling, TEACHER, dc), _config(modeling, student_cfg(n_student), dc)
    teacher = modeling.BertModel(t_conf)
    missing, unexpected = teacher.load_state_dict({k[len("bert."):]: v for k, v in teacher_params().items()}, strict=False)
    assert not missing and not unexpected, (missing, unexpected)
    teacher.make_teacher()
    student = modeling.BertForPreTraining(s_conf)
    missing, unexpected = student.load_state_dict(student_params(n_student), strict=False)
    assert not missing and not unexpected, (missing, unexpected)
    hs, ht = hooks.DistillHooks({"nn_module_names": []}), hooks.DistillHooks({"nn_module_names": []})
    student.register_forward_hook(hs.child_to_main_hook)
    teacher.register_forward_hook(ht.child_to_main_hook)
    student.train(); teacher.train()
    tl = losses_mod.TransformerLosses(s_conf, t_conf, torch.device("cpu"), types.SimpleNamespace(train_batch_size=B))
    b = distill_batch()
    student(b["input_ids"], b["token_type_ids"], b["attention_mask"], None)
    fs = hooks.flatten_states
    s_atts = fs(student.distill_states_dict, "attention_scores")
    s_reps = fs(student.distill_states_dict, "hidden_states")
    s_vals = fs(student.distill_states_dict, "value_states")
    s_embs = fs(student.distill_states_dict, "embedding_states")
    with torch.no_grad():
        teacher(b["input_ids"], b["token_type_ids"], b["attention_mask"])
    t_atts = [i.detach() for i in fs(teacher.distill_states_dict, "attention_scores")]
    t_reps = [i.detach() for i in fs(teacher.distill_states_dict, "hidden_states")]
    t_vals = [i.detach() for i in fs(teacher.distill_states_dict, "value_states")]
    t_embs = [i.detach() for i in fs(teacher.distill_states_dict, "embedding_states")]
    # general_distill.py:409-437, verbatim in substance
    if mapping == "last_layer":
        s_atts, n_t_atts = [s_atts[-1]], [t_atts[-1]]
        s_vals, n_t_vals = [s_vals[-1]], [t_vals[-1]]
        n_t_reps, n_s_reps = [t_reps[-1]], [s_reps[-1]]
    else:
        k = len(t_atts) // len(s_atts)
        n_t_atts = [t_atts[i * k + k - 1] for i in range(len(s_atts))]
        n_t_vals = [t_vals[i * k + k - 1] for i in range(len(s_atts))]
        n_t_reps = [t_reps[i * k + k - 1] for i in range(len(s_atts))]
        n_s_reps = s_reps
    att = tl.compute_loss(s_atts, n_t_atts, loss_name="attention_loss")
    rep = tl.compute_loss(n_s_reps, n_t_reps, loss_name="hidden_state_loss")
    if use_emb:
        rep = rep + tl.compute_loss(s_embs, t_embs, loss_name="embedding_state_loss")
    val = tl.compute_loss(s_vals, n_t_vals, loss_name="value_state_loss")
    return att, rep, val, student


def import_reference():
    sys.path.insert(0, HERE)
    from make_golden import REF, import_reference_modeling
    modeling = import_reference_modeling()
    sys.path.insert(0, os.path.join(REF, "distillation"))
    import hooks                 # the reference's distillation/hooks.py
    import losses                # the reference's distillation/losses.py
    return modeling, hooks, losses


def main():
    modeling, hooks, losses_mod = import_reference()
    torch.manual_seed(0)
    out = dict(batch=distill_batch(), cases=[])
    for n_student, mapping, use_emb in CASES:
        att, rep, val, student = reference_losses(modeling, hooks, losses_mod, n_student, mapping, use_emb)
        (att + rep + val).backward()
        grads = {k: p.grad.detach() for k, p in student.named_parameters() if p.grad is not None}
        out.setdefault("state_dict_keys", {})[n_student] = list(student.state_dict().keys())
        out["cases"].append(dict(n_student=n_student, mapping=mapping, use_embedding_states=use_emb, att_loss=att.detach(),
                                 rep_loss=rep.detach(), value_loss=val.detach(), grad_keys=list(grads),
                                 grad_norms=torch.stack([v.norm() for v in grads.values()]),
                                 grads_strided=torch.cat([v.reshape(-1)[::STRIDE] for v in grads.values()])))
        print(n_student, mapping, use_emb, "att", att.item(), "rep", rep.item(), "value", val.item(), "grads", len(grads))
    torch.save(out, os.path.join(HERE, "bert_distill_golden.pt"))


if __name__ == "__main__":
    main()
