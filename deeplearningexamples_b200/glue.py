"""GLUE fine-tuning step: the same encoder kernels under BertForSequenceClassification, with the reference step's structure
(PyTorch/LanguageModeling/BERT/run_glue.py):

    parameter groups with the pooler, no_decay = bias / LayerNorm.*                :298-316
    FusedAdam(lr, bias_correction=False) under amp O2, LinearWarmUpScheduler       :326-347  -> adam.FusedAdam (bf16 model + fp32 masters)
    loss = CrossEntropyLoss()(logits.view(-1, L), label_ids.view(-1)), ignore_index -100   :597,631-634
    loss.backward(); scheduler.step(); optimizer.step(); optimizer.zero_grad()       :642-657   (no gradient clipping)

Differences: bf16 instead of fp16 (no loss scaling needed; a GradScaler can still be passed), the schedule can live on the device
(CUDA-graph capturable), and the head's dropout is drawn from the device step counter like every other dropout mask.

Packed examples: with model.pack_sequences(k), glue_training_step and training.capture_step_graph take a packed GLUE batch
(packing.py: input_mask holds sample numbers, label_ids is [B*k] with -100 in empty slots) unchanged.  The logits are [B*k, L], one
row per sample slot, and the reference's loss line averages over the real samples, one term per example, as on padded rows.
"""
import numpy as np
import torch

from . import modeling
from .adam import FusedAdam
from .schedulers import LinearWarmUpScheduler


def glue_flops_per_seq(cfg, S):
    """3 x forward contractions of the encoder at sequence length S (the pooler and the classifier are negligible)."""
    L_, H, I = cfg["num_hidden_layers"], cfg["hidden_size"], cfg["intermediate_size"]
    return 3 * L_ * (6 * S * H * H + 4 * S * S * H + 2 * S * H * H + 4 * S * H * I)


def synthetic_glue_features(B, S, vocab, num_labels, seed=42, min_len=None, max_len=None):
    """A synthetic stand-in for a GLUE sentence-pair stream (no real GLUE data is read): an unpacked batch of right-padded rows
    (0/1 input_mask) that packing.PackedLoader(glue=True) also takes.  Lengths ~ U{min_len..max_len} (default U{S/8..S/2}); each row
    is [CLS] a [SEP] b [SEP] with segment 1 on b [SEP], and labels ~ U{0..num_labels-1}.  It makes no claim about the length
    distribution of any GLUE task."""
    min_len = max(5, S // 8) if min_len is None else min_len
    max_len = S // 2 if max_len is None else max_len
    if not 5 <= min_len <= max_len <= S:
        raise ValueError(f"lengths must satisfy 5 <= min_len <= max_len <= S, got {min_len}, {max_len}, S = {S}")
    g = torch.Generator().manual_seed(seed)
    lens = torch.randint(min_len, max_len + 1, (B,), generator=g)
    ids = torch.randint(1000, min(vocab, 30522), (B, S), generator=g, dtype=torch.int64)
    a_len = 1 + (torch.rand(B, generator=g) * (lens - 4).float()).long()          # 1..len-4 tokens of sentence a
    pos = torch.arange(S).unsqueeze(0)
    am = (pos < lens.unsqueeze(1)).to(torch.int64)
    sep_a = (a_len + 1).unsqueeze(1)
    ids[:, 0] = 101
    ids = torch.where(pos == sep_a, torch.full_like(ids, 102), ids)
    ids = torch.where(pos == (lens - 1).unsqueeze(1), torch.full_like(ids, 102), ids)
    ids *= am
    seg = ((pos > sep_a) & (am != 0)).to(torch.int64)
    labels = torch.randint(0, num_labels, (B,), generator=g, dtype=torch.int64)
    return {"input_ids": ids, "input_mask": am, "segment_ids": seg, "label_ids": labels}


def prepare_glue_model_and_optimizer(config_dict, device, num_labels, *, learning_rate=2.4e-5, warmup_proportion=0.1, total_steps=1000,
                                     dtype=torch.bfloat16, seed=42, device_schedule=True, state_dict=None):
    cfg = dict(config_dict)
    if cfg["vocab_size"] % 8 != 0:                                   # run_glue.py:553-554
        cfg["vocab_size"] += 8 - (cfg["vocab_size"] % 8)
    torch.manual_seed(seed)
    model = modeling.BertForSequenceClassification(modeling.BertConfig.from_dict(cfg), num_labels=num_labels)
    if state_dict is not None:
        model.load_state_dict(state_dict, strict=False)
    model.to(device).to(dtype)
    named = list(model.named_parameters())                           # the pooler is trained (:300)
    no_decay = ['bias', 'LayerNorm.bias', 'LayerNorm.weight']
    groups = [{'params': [p for n, p in named if not any(nd in n for nd in no_decay)], 'weight_decay': 0.01},
              {'params': [p for n, p in named if any(nd in n for nd in no_decay)], 'weight_decay': 0.0}]
    optimizer = FusedAdam(groups, lr=learning_rate, bias_correction=False, max_grad_norm=0.0)
    scheduler = LinearWarmUpScheduler(optimizer, warmup=warmup_proportion, total_steps=total_steps,
                                      device=device if device_schedule else None, base_lr=learning_rate)
    optimizer.setup_fp32_params()
    return model, optimizer, scheduler


def glue_loss(logits, label_ids):
    """run_glue.py:597,631-634: CrossEntropyLoss() (ignore_index -100) in fp32 on the bf16 logits."""
    return torch.nn.CrossEntropyLoss()(logits.float().view(-1, logits.shape[-1]), label_ids.view(-1))


def glue_training_step(model, optimizer, scheduler, batch, loss_acc=None, grad_scaler=None):
    """One iteration of the reference loop body (:628-657) with gradient_accumulation_steps = 1."""
    logits = model(batch["input_ids"], batch["segment_ids"], batch["input_mask"])
    loss = glue_loss(logits, batch["label_ids"])
    if loss_acc is not None:
        loss_acc.add_(loss.detach())
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
    return loss


def glue_predictions(logits, batch):
    """(example_index, predicted label) as host int64 arrays: over the non-empty slots of a packed batch (its example_index), or over
    every row of a padded batch (row numbers).  Metrics (accuracy, MCC, F1) are the caller's."""
    pred = logits.detach().argmax(-1).cpu().numpy()
    index = getattr(batch, "example_index", None)
    if index is None:
        return np.arange(pred.shape[0], dtype=np.int64), pred
    keep = index >= 0
    return index[keep], pred[keep]
