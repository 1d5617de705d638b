"""SWAG fine-tuning step: the same encoder kernels under BertForMultipleChoice, with the fp16 path of the reference step
(PyTorch/LanguageModeling/BERT/run_swag.py):

    parameter groups without the pooler, no_decay = bias / LayerNorm.*                  :406-416
    FusedAdam(lr, bias_correction=False, max_grad_norm=1.0) under FP16_Optimizer         :424-431  -> adam.FusedAdam (bf16 model + fp32 masters)
    loss = model(input_ids, segment_ids, input_mask, label_ids)  (the model's own CrossEntropyLoss)   :466-468
    lr = base * warmup_linear(global_step / t_total, warmup); optimizer.step(); zero_grad()          :481-494

Differences: bf16 instead of fp16 (no loss scaling needed; a GradScaler can still be passed), the schedule can live on the device
(CUDA-graph capturable), the head's dropout is drawn from the device step counter like every other dropout mask, and the pooler's
parameters are frozen with requires_grad_(False).  The reference leaves the pooler out of the optimizer but still computes its
gradients (the head reads the pooled output); here none are computed, so nothing accumulates into a .grad no optimizer clears.

The reference's schedule runs at progress global_step / t_total, so its first step runs at lr 0: LinearWarmUpScheduler with
progress_offset=0 (SQuAD and GLUE use (step + 1) / total).

Packed examples: with model.pack_sequences(k), k a multiple of num_choices, swag_training_step and training.capture_step_graph take a
packed SWAG batch (packing.py: input_mask holds sample numbers, one per choice, label_ids is [B*k/C] with -100 in empty groups)
unchanged.  The model's view(-1, C) turns the [B*k, 1] scores into one row per group of C slots, and the loss averages over the real
examples, one term per example, as on padded batches.
"""
import numpy as np
import torch

from . import modeling
from .adam import FusedAdam
from .glue import glue_flops_per_seq
from .schedulers import LinearWarmUpScheduler


def swag_flops_per_example(cfg, S, num_choices=4):
    """3 x forward contractions of the encoder over an example's num_choices rows of S tokens (the pooler and the classifier are
    negligible): the work a padded step spends per example."""
    return num_choices * glue_flops_per_seq(cfg, S)


def warmup_linear(x, warmup=0.002):
    """optimization.py:46-49, the reference's schedule factor at progress x."""
    if x < warmup:
        return x / warmup
    return max((x - 1.) / (warmup - 1.), 0.)


def synthetic_swag_features(N, C, S, vocab, seed=42, min_context=None, max_context=None, min_ending=None, max_ending=None):
    """A synthetic stand-in for a SWAG example stream (no real SWAG data is read), laid out as run_swag.py's
    convert_examples_to_features lays it out (:139-190): input_ids, input_mask, segment_ids [N, C, S], label_ids [N].  Choice c of an
    example is [CLS] context [SEP] ending_c [SEP], right-padded to S, with segment 0 through the first [SEP] and 1 after it; the same
    context appears in all C choices, each with its own ending.  Context lengths ~ U{min_context..max_context} (default U{S/16..S/4})
    and ending lengths ~ U{min_ending..max_ending} (default U{S/32..S/8}) tokens; labels ~ U{0..C-1}.  It makes no claim about the
    length distribution of the real SWAG data."""
    min_context = max(1, S // 16) if min_context is None else min_context
    max_context = S // 4 if max_context is None else max_context
    min_ending = max(1, S // 32) if min_ending is None else min_ending
    max_ending = S // 8 if max_ending is None else max_ending
    if not (1 <= min_context <= max_context and 1 <= min_ending <= max_ending and max_context + max_ending + 3 <= S):
        raise ValueError(f"lengths must satisfy 1 <= min <= max and max_context + max_ending + 3 <= S, got context "
                         f"{min_context}..{max_context}, ending {min_ending}..{max_ending}, S = {S}")
    rng = np.random.default_rng(seed)
    hi = min(vocab, 30522)
    ids = np.zeros((N, C, S), np.int64)
    seg = np.zeros((N, C, S), np.int64)
    am = np.zeros((N, C, S), np.int64)
    for n in range(N):
        a = int(rng.integers(min_context, max_context + 1))
        context = rng.integers(1000, hi, a)
        for c in range(C):
            e = int(rng.integers(min_ending, max_ending + 1))
            row = np.concatenate([[101], context, [102], rng.integers(1000, hi, e), [102]])
            ids[n, c, :len(row)] = row
            am[n, c, :len(row)] = 1
            seg[n, c, a + 2:len(row)] = 1
    labels = rng.integers(0, C, N)
    return {key: torch.from_numpy(v) for key, v in
            (("input_ids", ids), ("input_mask", am), ("segment_ids", seg), ("label_ids", labels.astype(np.int64)))}


def prepare_swag_model_and_optimizer(config_dict, device, num_choices=4, *, learning_rate=5e-5, warmup_proportion=0.1, total_steps,
                                     dtype=torch.bfloat16, seed=42, device_schedule=True, state_dict=None):
    cfg = dict(config_dict)
    if cfg["vocab_size"] % 8 != 0:                                   # as glue / squad do, so their checkpoints load unchanged
        cfg["vocab_size"] += 8 - (cfg["vocab_size"] % 8)
    torch.manual_seed(seed)
    model = modeling.BertForMultipleChoice(modeling.BertConfig.from_dict(cfg), num_choices=num_choices)
    if state_dict is not None:
        model.load_state_dict(state_dict, strict=False)
    model.to(device).to(dtype)
    named = [(n, p) for n, p in model.named_parameters() if 'pooler' not in n]       # :408-410
    for n, p in model.named_parameters():
        if 'pooler' in n:
            p.requires_grad_(False)
    no_decay = ['bias', 'LayerNorm.bias', 'LayerNorm.weight']
    groups = [{'params': [p for n, p in named if not any(nd in n for nd in no_decay)], 'weight_decay': 0.01},
              {'params': [p for n, p in named if any(nd in n for nd in no_decay)], 'weight_decay': 0.0}]
    optimizer = FusedAdam(groups, lr=learning_rate, bias_correction=False, max_grad_norm=1.0)
    scheduler = LinearWarmUpScheduler(optimizer, warmup=warmup_proportion, total_steps=total_steps,
                                      device=device if device_schedule else None, base_lr=learning_rate, progress_offset=0)
    optimizer.setup_fp32_params()
    return model, optimizer, scheduler


def swag_training_step(model, optimizer, scheduler, batch, loss_acc=None, grad_scaler=None):
    """One iteration of the reference loop body (:466-494) with gradient_accumulation_steps = 1, on a padded ([B, C, S]) or packed
    ([B, S], model.pack_sequences(k)) batch."""
    loss = model(batch["input_ids"], batch["segment_ids"], batch["input_mask"], batch["label_ids"])
    if loss_acc is not None:
        loss_acc.add_(loss.detach())
    if grad_scaler is not None and grad_scaler.is_enabled():
        grad_scaler.scale(loss).backward()
        scheduler.step()
        grad_scaler.step(optimizer)
        grad_scaler.update()
    else:
        loss.backward()
        scheduler.step()            # lr = base * warmup_linear(global_step / t_total) (:486-491)
        optimizer.step()            # global-norm clip (max_grad_norm = 1.0) + Adam in one call
    optimizer.zero_grad(set_to_none=True)
    return loss


def swag_predictions(logits, batch):
    """(example_index, predicted choice) as host int64 arrays from the [groups, C] logits: over the non-empty groups of a packed batch
    (its example_index), or over every example of a padded batch (row numbers).  Accuracy (run_swag.py:233-235) is the caller's."""
    pred = logits.detach().argmax(-1).cpu().numpy()
    index = getattr(batch, "example_index", None)
    if index is None:
        return np.arange(pred.shape[0], dtype=np.int64), pred
    keep = index >= 0
    return index[keep], pred[keep]
