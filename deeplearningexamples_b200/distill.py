"""General (backbone) distillation on the fused encoder: the step of PyTorch/LanguageModeling/BERT/distillation/general_distill.py.

    teacher = BertModel.from_pretrained(..., distill_config); make_teacher()              :254-260
    student = BertForPreTraining.from_scratch / from_pretrained(..., distill_config)      :262-266  (no cls heads, no pooler)
    project = Project(student_config, teacher_config) when the widths differ              :268-276
    FusedAdam(bias_correction=False), two weight-decay groups, LinearWarmUpScheduler      :310-323
    states -> layer mapping -> att + rep + value losses -> clip(1.0) -> step              :378-489

The losses are the reference's (distillation/losses.py) without its [B, A, S, S] tensors: an attention-score pair is a pair of
modeling.AttentionScores handles and goes to the relation-KL kernel with X = Q, Y = K; a value-state pair goes to the same kernel with
X = Y = ctx; a cosine pair goes to the cosine-rows kernel.  Everything stays on the device: the step returns device tensors and can be
captured with training.capture_step_graph.

Not built (each raises DleError naming the config key): "mse" losses, a "cosine" attention or value loss, student / teacher head
counts or sequence lengths that differ, head size other than 64, and distillation together with remove_padding or pack_sequences.
"""
import logging
import math
from collections import OrderedDict

import torch

from . import _lib as L
from . import modeling
from . import ops
from .adam import FusedAdam
from .schedulers import LinearWarmUpScheduler


class DistillHooks:
    """distillation/hooks.py:17-96.  child_to_main_hook, registered as a forward hook on the top model, gathers every submodule's
    distill_state_dict into model.distill_states_dict (module name -> states)."""

    def __init__(self, config):
        self.nn_module_names = config["nn_module_names"]
        self.nn_module_states = {}

    def nn_module_hook(self, name):
        def hook(module, input, output):
            self.nn_module_states[name] = output
        return hook

    def register_nn_module_hook(self, module, input):
        for name, i in module.named_modules():
            if name in self.nn_module_names:
                i.register_forward_hook(self.nn_module_hook(name))

    def child_to_main_hook(self, module, input, output):
        module.distill_states_dict = OrderedDict()
        for name, i in module.named_modules():
            if hasattr(i, 'distill_state_dict'):
                module.distill_states_dict[name] = i.distill_state_dict


def flatten_states(state_dict, state_name):
    """hooks.py:99-108: the `state_name` entries of every module's states, in module order."""
    return [value[state_name] for value in state_dict.values() if state_name in value]


class TransformerLosses:
    """distillation/losses.py:21-88 on the fused kernels.  compute_loss(pred, target, loss_name) sums the pair losses."""

    def __init__(self, student_config, teacher_config, device, args):
        self.distill_config = student_config.distillation_config
        self.device = device
        self.student_config = student_config
        self.teacher_config = teacher_config
        self.batch_size = args.train_batch_size if args is not None and hasattr(args, "train_batch_size") else None
        check_distill_configs(student_config, teacher_config)

    def compute_loss_(self, pred, target, loss_name):
        kind = self.distill_config[loss_name]
        if kind == "kld":
            if loss_name == "attention_loss":
                return _attention_kl(pred, target)
            if loss_name == "value_state_loss":
                return _value_kl(pred, target)
            raise L.DleError(f"{loss_name}: 'kld' is defined for attention_loss and value_state_loss only")
        if kind == "cosine":
            if loss_name in ("attention_loss", "value_state_loss"):
                raise L.DleError(f"{loss_name}: 'cosine' is not built on the fused path (it needs the [B, A, S, S] tensors); use 'kld'")
            H = self.teacher_config.hidden_size
            x, y = _rows(pred, H), _rows(target, H)
            return ops.CosineRowsFn.apply(x, y)
        if kind == "mse":
            raise L.DleError(f"{loss_name}: 'mse' losses are not built on the fused path")
        raise ValueError("'{}':{} not defined. Choose among 'mse', 'cosine' or 'kld'".format(loss_name, kind))

    def compute_loss(self, pred, target, loss_name):
        loss = None
        for student, teacher in zip(pred, target):
            term = self.compute_loss_(student, teacher, loss_name)      # the where rule of :80-85 runs inside the kernel
            loss = term if loss is None else loss + term
        return torch.zeros((), device=self.device) if loss is None else loss


def _attention_kl(s, t):
    if not isinstance(s, modeling.AttentionScores) or not isinstance(t, modeling.AttentionScores):
        raise L.DleError("attention_loss 'kld' takes the AttentionScores handles the fused layers record")
    if (s.B, s.S, s.A) != (t.B, t.S, t.A) or s.seq_first != t.seq_first:
        raise L.DleError(f"attention_loss: student scores {tuple(s.shape)} and teacher scores {tuple(t.shape)} differ "
                         "(num_attention_heads and the sequence length must match)")
    cfg = ("attention", s.B, s.S, s.A, s.seq_first, s.mask, t.mask, s.scale, t.scale)
    return ops.RelationKLFn.apply(s.qkv, t.qkv.detach(), cfg)


def _value_kl(s, t):
    """value_states [S, B, A*64] of student and teacher: per (b, h) KL of softmax(V V^T / sqrt(d)) (losses.py:41-61)."""
    S, B, Hs = s.shape
    if tuple(t.shape[:2]) != (S, B):
        raise L.DleError(f"value_state_loss: student states {tuple(s.shape)} and teacher states {tuple(t.shape)} differ in length")
    if Hs % 64 != 0 or t.shape[2] % 64 != 0 or Hs != t.shape[2]:
        raise L.DleError("value_state_loss: student and teacher need the same number of heads of size 64 "
                         f"(hidden {Hs} and {t.shape[2]})")
    xs, _, tr_s = modeling._tokens(s)
    xt, _, tr_t = modeling._tokens(t.detach())
    if tr_s != tr_t:
        raise L.DleError("value_state_loss: student and teacher states are in different token orders")
    A = Hs // 64
    scale = 1.0 / math.sqrt(64)
    cfg = ("value", B, S, A, not tr_s, None, None, scale, scale)
    return ops.RelationKLFn.apply(xs, xt, cfg)


def _rows(x, H):
    """[rows, H] bf16 view of a state tensor in its memory order (student and teacher states share it)."""
    x2, _, _ = modeling._tokens(x)
    if x2.shape[1] != H:
        raise L.DleError(f"cosine loss: states of width {x2.shape[1]}, expected the teacher's hidden size {H}")
    return x2


def check_distill_configs(student_config, teacher_config):
    """Refuse what the fused path does not build, naming the config key."""
    dc = student_config.distillation_config
    for key in ("attention_loss", "value_state_loss", "hidden_state_loss", "embedding_state_loss"):
        if dc.get(key) == "mse":
            raise L.DleError(f"{key}: 'mse' losses are not built on the fused path")
    for key in ("attention_loss", "value_state_loss"):
        if dc.get(key) == "cosine":
            raise L.DleError(f"{key}: 'cosine' is not built on the fused path; use 'kld'")
    if dc.get("use_attention_scores") or dc.get("use_value_states"):
        if student_config.num_attention_heads != teacher_config.num_attention_heads:
            raise L.DleError(f"num_attention_heads: student {student_config.num_attention_heads} and teacher "
                             f"{teacher_config.num_attention_heads} differ (the relation losses pair heads one to one)")
    for name, c in (("student", student_config), ("teacher", teacher_config)):
        if c.hidden_size // c.num_attention_heads != 64 or c.hidden_size % c.num_attention_heads != 0:
            raise L.DleError(f"hidden_size / num_attention_heads: the {name}'s head size is "
                             f"{c.hidden_size / c.num_attention_heads:g}; the fused kernels take 64")


def _layer_map(n_student, n_teacher, mapping):
    """Teacher layer index for each student layer (general_distill.py:409-437)."""
    if mapping == "last_layer":
        return None
    if n_teacher % n_student != 0:
        raise L.DleError(f"student_teacher_layer_mapping: {n_teacher} teacher layers are not a multiple of {n_student} student layers")
    k = n_teacher // n_student
    return [i * k + k - 1 for i in range(n_student)]


def distill_losses(student, teacher, project, losses, batch):
    """Forward of both models and the three losses of general_distill.py:380-467: (att_loss, rep_loss, value_loss), 0-d device
    tensors (zero for a disabled term)."""
    input_ids, segment_ids, input_mask = batch["input_ids"], batch["token_type_ids"], batch["attention_mask"]
    for m in (student, teacher):
        if getattr(_bert(m), "_remove_padding", False) or getattr(_bert(m), "_pack_per_row", 0):
            raise L.DleError("distillation with remove_padding or pack_sequences is not built: turn both routes off")
    student(input_ids, segment_ids, input_mask, None)
    s_states = student.distill_states_dict
    with torch.no_grad():
        teacher(input_ids, segment_ids, input_mask)
    t_states = teacher.distill_states_dict
    dc = losses.student_config.distillation_config
    dev = input_ids.device
    zero = torch.zeros((), device=dev, dtype=torch.float32)

    s_atts, t_atts = flatten_states(s_states, "attention_scores"), [i.detach() for i in flatten_states(t_states, "attention_scores")]
    s_reps, t_reps = flatten_states(s_states, "hidden_states"), [i.detach() for i in flatten_states(t_states, "hidden_states")]
    s_vals, t_vals = flatten_states(s_states, "value_states"), [i.detach() for i in flatten_states(t_states, "value_states")]
    s_embs, t_embs = flatten_states(s_states, "embedding_states"), [i.detach() for i in flatten_states(t_states, "embedding_states")]
    n_s = losses.student_config.num_hidden_layers
    n_t = losses.teacher_config.num_hidden_layers
    idx = _layer_map(n_s, n_t, dc["student_teacher_layer_mapping"])
    pick = (lambda s, t: ([s[-1]], [t[-1]])) if idx is None else (lambda s, t: (s, [t[i] for i in idx]))

    att_loss = rep_loss = value_loss = zero
    if dc["use_attention_scores"]:
        att_loss = losses.compute_loss(*pick(s_atts, t_atts), loss_name="attention_loss")
    if dc["use_hidden_states"]:
        sr, tr = pick(s_reps, t_reps)
        rep_loss = losses.compute_loss(project(sr) if project is not None else sr, tr, loss_name="hidden_state_loss")
    if dc["use_embedding_states"]:
        rep_loss = rep_loss + losses.compute_loss(project(s_embs) if project is not None else s_embs, t_embs,
                                                  loss_name="embedding_state_loss")
    if dc["use_value_states"]:
        value_loss = losses.compute_loss(*pick(s_vals, t_vals), loss_name="value_state_loss")
    return att_loss, rep_loss, value_loss


def _bert(m):
    return getattr(m, "bert", m)


def general_distill_step(student, teacher, project, losses, optimizer, scheduler, batch, grad_scaler=None):
    """One iteration of general_distill.py:378-489 with gradient_accumulation_steps = 1: both forwards, loss = att + rep + value,
    backward, scheduler.step() before the optimizer step (global-norm clip at 1.0 over student and Project inside FusedAdam).
    Returns (loss, att_loss, rep_loss, value_loss) as device tensors; nothing is read on the host."""
    att_loss, rep_loss, value_loss = distill_losses(student, teacher, project, losses, batch)
    loss = att_loss + rep_loss + value_loss
    if grad_scaler is not None and grad_scaler.is_enabled():
        grad_scaler.scale(loss).backward()
        scheduler.step()
        grad_scaler.step(optimizer)
        grad_scaler.update()
    else:
        loss.backward()
        scheduler.step()
        optimizer.step()
    optimizer.zero_grad(set_to_none=True)
    return loss.detach(), att_loss.detach(), rep_loss.detach(), value_loss.detach()


def _load(model, state_dict, what):
    """load_state_dict(strict=False), as from_pretrained loads (a pretraining checkpoint carries pooler / cls keys a distillation model
    does not have), with the key mismatches reported: a missing key leaves that parameter at its random initialisation."""
    result = model.load_state_dict(state_dict, strict=False)
    log = logging.getLogger(__name__)
    if result.missing_keys:
        log.warning("%s: weights not initialized from the state dict: %s", what, result.missing_keys)
    if result.unexpected_keys:
        log.info("%s: weights from the state dict not used: %s", what, result.unexpected_keys)
    return result


def prepare_distill_models_and_optimizer(student_cfg, teacher_cfg, device, distill_config, *, learning_rate=5e-5,
                                         warmup_proportion=0.01, total_steps, dtype=torch.bfloat16, seed=42, device_schedule=True,
                                         teacher_state_dict=None, student_state_dict=None, project_state_dict=None):
    """general_distill.py:254-323 from config dicts: (student, teacher, project or None, losses, optimizer, scheduler).  The teacher is a
    BertModel with make_teacher(); the student a BertForPreTraining without heads; both carry `distill_config` (a dict or JSON path).
    Forward hooks gather their states as the reference's DistillHooks do.  The teacher's train / eval mode is the caller's: the reference
    never puts it in eval mode, so its dropout is on in training."""
    torch.manual_seed(seed)
    s_cfg, t_cfg = modeling.BertConfig.from_dict(dict(student_cfg)), modeling.BertConfig.from_dict(dict(teacher_cfg))
    modeling._apply_distill_config(t_cfg, distill_config, True)
    modeling._apply_distill_config(s_cfg, distill_config, True)
    check_distill_configs(s_cfg, t_cfg)
    teacher = modeling.BertModel(t_cfg)
    if teacher_state_dict is not None:
        _load(teacher, teacher_state_dict, "teacher")
    teacher.make_teacher()
    student = modeling.BertForPreTraining(s_cfg)
    if student_state_dict is not None:
        _load(student, student_state_dict, "student")
    project = modeling.Project(s_cfg, t_cfg) if s_cfg.hidden_size != t_cfg.hidden_size else None
    if project is not None and project_state_dict is not None:
        project.load_state_dict(project_state_dict)
    hooks_s, hooks_t = DistillHooks({"nn_module_names": []}), DistillHooks({"nn_module_names": []})
    student.register_forward_hook(hooks_s.child_to_main_hook)
    teacher.register_forward_hook(hooks_t.child_to_main_hook)
    for m in (student, teacher, project):
        if m is not None:
            m.to(device).to(dtype)
    named = list(student.named_parameters()) + (list(project.named_parameters()) if project is not None else [])
    no_decay = ['bias', 'LayerNorm.bias', 'LayerNorm.weight']
    groups = [{'params': [p for n, p in named if not any(nd in n for nd in no_decay)], 'weight_decay': 0.01},
              {'params': [p for n, p in named if any(nd in n for nd in no_decay)], 'weight_decay': 0.0}]
    optimizer = FusedAdam(groups, lr=learning_rate, bias_correction=False, max_grad_norm=1.0)
    scheduler = LinearWarmUpScheduler(optimizer, warmup=warmup_proportion, total_steps=total_steps,
                                      device=device if device_schedule else None, base_lr=learning_rate)
    optimizer.setup_fp32_params()
    losses = TransformerLosses(s_cfg, t_cfg, device, None)
    return student, teacher, project, losses, optimizer, scheduler

