"""SQuAD fine-tuning step (BASELINE.json configs[3]; SURVEY.md 8f rank 1): the same encoder kernels at seq 384 under a QA head, with
the reference step's structure (PyTorch/LanguageModeling/BERT/run_squad.py):

    parameter groups without the pooler, no_decay = bias / LayerNorm.*        :955-964
    FusedAdam(lr, bias_correction=False) under amp O2 (16-bit model, fp32 masters)  :969-975  -> adam.FusedAdam (bf16 model + fp32 masters)
    loss = (CE(start_logits, start) + CE(end_logits, end)) / 2, positions clamped to [0, S], ignore_index = S   :1062-1071
    GradientClipper(max_grad_norm=1.0): coef = max / (norm + 1e-6) applied when < 1     :703-724,1089  -> fused into dle_adam_step
    LinearWarmUpScheduler.step(); optimizer.step(); optimizer.zero_grad()            :1091-1098

Differences: bf16 instead of fp16 (no loss scaling needed; a GradScaler can still be passed), the clip is part of the optimizer
launch instead of a separate l2norm + scale sweep, the schedule can live on the device (CUDA-graph capturable).

Packed features: with model.pack_sequences(k, per_sample_logits=True), squad_training_step and training.capture_step_graph take a
packed SQuAD batch (packing.py: input_mask holds sample numbers, start/end_positions are [B*k], one per sample slot, S in an empty
slot) unchanged.  The logits are [B*k, S], each sample's own positions first and BertForQuestionAnswering.SPAN_FILL after them, so
squad_loss clamps to [0, S] and ignores S exactly as on padded rows.  A sample's cross-entropy then runs over its own len positions:
it equals the padded route's on the same feature with the logits of its padding positions set to SPAN_FILL (the padded route also
softmaxes over its padding logits).  The mean runs over the counted slots, one term per feature, as the reference's does.
"""
import torch

from . import modeling
from .adam import FusedAdam
from .schedulers import LinearWarmUpScheduler


def squad_flops_per_seq(cfg, S):
    """3 x forward contractions of the encoder (QA head and pooler are negligible), SURVEY.md 8d: 739.3 GF at S=384 for BERT-large."""
    L_, H, I = cfg["num_hidden_layers"], cfg["hidden_size"], cfg["intermediate_size"]
    return 3 * L_ * (6 * S * H * H + 4 * S * S * H + 2 * S * H * H + 4 * S * H * I)


def synthetic_squad_batch(B, S, vocab, seed=42, full_mask=True, device="cpu", pin=False):
    """SURVEY.md 8d config (4): ids ~ U{0..30521}, segment split, start/end positions ~ U{0..S-1}."""
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(0, min(vocab, 30522), (B, S), generator=g, dtype=torch.int64)
    ids[:, 0] = 101
    seg = torch.zeros(B, S, dtype=torch.int64)
    seg[:, S // 4:] = 1
    if full_mask:
        am = torch.ones(B, S, dtype=torch.int64)
    else:
        lens = torch.randint(S // 4, S + 1, (B,), generator=g)
        am = (torch.arange(S).unsqueeze(0) < lens.unsqueeze(1)).to(torch.int64)
    start = torch.randint(0, S, (B,), generator=g, dtype=torch.int64)
    end = torch.randint(0, S, (B,), generator=g, dtype=torch.int64)
    batch = {"input_ids": ids, "input_mask": am, "segment_ids": seg, "start_positions": start, "end_positions": end}
    if pin:
        batch = {k: v.pin_memory() for k, v in batch.items()}
    if device != "cpu":
        batch = {k: v.to(device) for k, v in batch.items()}
    return batch


def synthetic_squad_features(B, S, vocab, seed=42):
    """Variable-length SQuAD features as an unpacked batch (right-padded rows, 0/1 input_mask) that packing.PackedLoader(squad=True)
    also takes: lengths ~ U{S/4..S} as synthetic_squad_batch(full_mask=False), [CLS] first, segment 1 on the last three quarters of
    each feature, and an answer span inside it (start ~ U{0..len-1}, end ~ U{start..len-1})."""
    g = torch.Generator().manual_seed(seed)
    lens = torch.randint(S // 4, S + 1, (B,), generator=g)
    ids = torch.randint(0, min(vocab, 30522), (B, S), generator=g, dtype=torch.int64)
    ids[:, 0] = 101
    pos = torch.arange(S).unsqueeze(0)
    am = (pos < lens.unsqueeze(1)).to(torch.int64)
    ids *= am
    seg = ((pos >= (lens // 4).unsqueeze(1)) & (am != 0)).to(torch.int64)
    start = (torch.rand(B, generator=g) * lens).long()
    end = start + (torch.rand(B, generator=g) * (lens - start)).long()
    return {"input_ids": ids, "input_mask": am, "segment_ids": seg, "start_positions": start, "end_positions": end}


def prepare_squad_model_and_optimizer(config_dict, device, *, learning_rate=3e-5, warmup_proportion=0.1, total_steps=1000,
                                      dtype=torch.bfloat16, seed=42, distributed=False, device_schedule=True, state_dict=None):
    cfg = dict(config_dict)
    if cfg["vocab_size"] % 8 != 0:                                   # run_squad.py:935-936
        cfg["vocab_size"] += 8 - (cfg["vocab_size"] % 8)
    torch.manual_seed(seed)
    model = modeling.BertForQuestionAnswering(modeling.BertConfig.from_dict(cfg))
    if state_dict is not None:
        model.load_state_dict(state_dict, strict=False)              # run_squad.py:941-944 (init_checkpoint, strict=False)
    model.to(device).to(dtype)
    named = [(n, p) for n, p in model.named_parameters() if 'pooler' not in n]       # :958-959 (the QA model never uses the pooler)
    for n, p in model.named_parameters():
        if 'pooler' in n:
            p.requires_grad_(False)
    no_decay = ['bias', 'LayerNorm.bias', 'LayerNorm.weight']
    groups = [{'params': [p for n, p in named if not any(nd in n for nd in no_decay)], 'weight_decay': 0.01},
              {'params': [p for n, p in named if any(nd in n for nd in no_decay)], 'weight_decay': 0.0}]
    optimizer = FusedAdam(groups, lr=learning_rate, bias_correction=False, max_grad_norm=1.0)
    scheduler = LinearWarmUpScheduler(optimizer, warmup=warmup_proportion, total_steps=total_steps,
                                      device=device if device_schedule else None, base_lr=learning_rate)
    if distributed:
        from torch.nn.parallel import DistributedDataParallel as DDP
        side = torch.cuda.Stream()
        with torch.cuda.stream(side):
            model = DDP(model, device_ids=[device.index], output_device=device.index, bucket_cap_mb=100, gradient_as_bucket_view=True)
        torch.cuda.current_stream().wait_stream(side)
    optimizer.setup_fp32_params()
    return model, optimizer, scheduler


def squad_loss(start_logits, end_logits, start_positions, end_positions):
    """run_squad.py:1062-1071; cross-entropy in fp32 on the bf16 logits."""
    ignored_index = start_logits.size(1)
    sp = start_positions.clamp(0, ignored_index)
    ep = end_positions.clamp(0, ignored_index)
    loss_fct = torch.nn.CrossEntropyLoss(ignore_index=ignored_index)
    return (loss_fct(start_logits.float(), sp) + loss_fct(end_logits.float(), ep)) / 2


def squad_training_step(model, optimizer, scheduler, batch, loss_acc=None, grad_scaler=None):
    """One iteration of the reference loop body (:1051-1098) with gradient_accumulation_steps = 1."""
    start_logits, end_logits = model(batch["input_ids"], batch["segment_ids"], batch["input_mask"])
    loss = squad_loss(start_logits, end_logits, batch["start_positions"], batch["end_positions"])
    if loss_acc is not None:
        loss_acc.add_(loss.detach())
    if grad_scaler is not None and grad_scaler.is_enabled():
        grad_scaler.scale(loss).backward()
        scheduler.step()
        grad_scaler.step(optimizer)
        grad_scaler.update()
    else:
        loss.backward()
        scheduler.step()            # "modify learning rate with special warm up for BERT which FusedAdam doesn't do" (:1092-1094)
        optimizer.step()            # global-norm clip (GradientClipper, :1089) + Adam in one call
    optimizer.zero_grad(set_to_none=True)
    return loss
