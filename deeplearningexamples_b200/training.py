"""Training-step glue mirroring the reference driver's functions
(PyTorch/LanguageModeling/BERT/run_pretraining.py) so bench.py, smoke() and the tests execute the same
sequence the reference's main loop does:

  BertPretrainingCriterion   run_pretraining.py:75-95
  prepare_model_and_optimizer  :377-486  (param groups :422-427, FusedLAMBAMP :429, scheduler :431-435,
                                          GradScaler :436, DDP wrap :455-458, setup_fp32_params :477)
  take_training_step         :518-524
  take_optimizer_step        :527-536
  synthetic_batch            the lddl batch format read at :520-521,603-609 (five int64 tensors)

Differences: bf16 instead of fp16 (`model.bfloat16()` where the reference does `model.half()` for
--allreduce_post_accumulation_fp16); DDP uses overlap-sized buckets instead of one bucket of total_memory MB.
"""
import torch

from . import modeling, ops
from .lamb import FusedLAMBAMP
from .schedulers import PolyWarmUpScheduler

BERT_LARGE = dict(attention_probs_dropout_prob=0.1, hidden_act="gelu", hidden_dropout_prob=0.1, hidden_size=1024,
                  initializer_range=0.02, intermediate_size=4096, max_position_embeddings=512, num_attention_heads=16,
                  num_hidden_layers=24, type_vocab_size=2, vocab_size=30522)
BERT_BASE = dict(attention_probs_dropout_prob=0.1, hidden_act="gelu", hidden_dropout_prob=0.1, hidden_size=768,
                 initializer_range=0.02, intermediate_size=3072, max_position_embeddings=512, num_attention_heads=12,
                 num_hidden_layers=12, type_vocab_size=2, vocab_size=30528)

# training FLOPs per sequence (SURVEY.md 8d): 3 x forward, GEMM + attention contractions only
def train_flops_per_seq(cfg, S, P):
    L_, H, I, V = cfg["num_hidden_layers"], cfg["hidden_size"], cfg["intermediate_size"], cfg["vocab_size"]
    fwd = L_ * (6 * S * H * H + 4 * S * S * H + 2 * S * H * H + 4 * S * H * I) + (2 * P * H * H + 2 * P * H * V + 2 * H * H)
    return 3 * fwd


class BertPretrainingCriterion(torch.nn.Module):
    def __init__(self, vocab_size, sequence_output_is_dense=False):
        super().__init__()
        self.loss_fn = torch.nn.CrossEntropyLoss(ignore_index=-1)
        self.vocab_size = vocab_size
        self.sequence_output_is_dense = sequence_output_is_dense
        self.fused_ce = True

    def forward(self, prediction_scores, seq_relationship_score, masked_lm_labels, next_sentence_labels):
        # cross-entropy runs in fp32 on the bf16 logits, as it does under the reference's autocast (CE is on autocast's fp32 list;
        # run_pretraining.py:519-522).  CUDA bf16 logits take the fused kernel (fp32 arithmetic in registers, no fp32 copy of the
        # [rows, V] tensor: ops.SoftmaxCrossEntropyFn); anything else goes through torch on an fp32 copy.
        scores = prediction_scores.view(-1, self.vocab_size)
        fused = self.fused_ce and scores.is_cuda and scores.dtype == torch.bfloat16 and self.vocab_size % 8 == 0 and self.vocab_size <= 32768
        if not fused:
            scores = scores.float()
        mlm_loss_fn = (lambda sc, lab: ops.SoftmaxCrossEntropyFn.apply(sc, lab, -1)) if fused else self.loss_fn
        if self.sequence_output_is_dense:
            # reference: labels[labels != -1] (boolean indexing => host sync).  Same rows, same order, without the sync: the
            # first `n` non-ignored positions, n = rows of the (already dense) prediction scores; surplus slots (static-count
            # mode, index -1) get label -1 and are ignored by the loss.
            flat = masked_lm_labels.view(-1)
            idx = torch.nonzero_static(flat != -1, size=scores.shape[0], fill_value=-1).squeeze(-1)
            mlm_labels = torch.where(idx >= 0, flat[idx.clamp_min(0)], torch.full_like(idx, -1))
            masked_lm_loss = mlm_loss_fn(scores, mlm_labels)
        else:
            masked_lm_loss = mlm_loss_fn(scores, masked_lm_labels.view(-1))
        next_sentence_loss = self.loss_fn(seq_relationship_score.view(-1, 2).float(), next_sentence_labels.view(-1))
        return masked_lm_loss + next_sentence_loss


def synthetic_batch(B, S, vocab, max_pred, seed=42, full_mask=True, device="cpu", pin=False):
    """SURVEY.md 8(d): ids ~ U{0..30521} with [CLS] first, segment split at S/2, exactly max_pred labels per row."""
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(0, min(vocab, 30522), (B, S), generator=g, dtype=torch.int64)
    ids[:, 0] = 101
    tt = torch.zeros(B, S, dtype=torch.int64)
    tt[:, S // 2:] = 1
    if full_mask:
        am = torch.ones(B, S, dtype=torch.int64)
    else:
        lens = (torch.randint(S // 4, S + 1, (B,), generator=g) + 63) // 64 * 64
        am = (torch.arange(S).unsqueeze(0) < lens.clamp(max=S).unsqueeze(1)).to(torch.int64)
    labels = torch.full((B, S), -1, dtype=torch.int64)
    for b in range(B):
        pos = torch.randperm(S, generator=g)[:max_pred]
        labels[b, pos] = torch.randint(0, min(vocab, 30522), (max_pred,), generator=g)
    nsl = torch.randint(0, 2, (B,), generator=g, dtype=torch.int64)
    batch = {"input_ids": ids, "token_type_ids": tt, "attention_mask": am, "labels": labels, "next_sentence_labels": nsl}
    if pin:
        batch = {k: v.pin_memory() for k, v in batch.items()}
    if device != "cpu":
        batch = {k: v.to(device) for k, v in batch.items()}
    return batch


def prepare_model_and_optimizer(config_dict, device, *, learning_rate=6e-3, warmup_proportion=0.2843, max_steps=7038,
                                sequence_output_is_dense=True, init_loss_scale=2 ** 20, use_grad_scaler=True,
                                distributed=False, bucket_cap_mb=100, dtype=torch.bfloat16, seed=42, static_masked_count=None):
    cfg = dict(config_dict)
    if cfg["vocab_size"] % 8 != 0:                       # run_pretraining.py:383-384
        cfg["vocab_size"] += 8 - (cfg["vocab_size"] % 8)
    config = modeling.BertConfig.from_dict(cfg)
    torch.manual_seed(seed)
    model = modeling.BertForPreTraining(config, sequence_output_is_dense=sequence_output_is_dense)
    if static_masked_count:
        model.cls.static_masked_count = int(static_masked_count)
    model.to(device)
    model.to(dtype)                                       # the reference's model.half() (:416-417), in bf16
    no_decay = ['bias', 'gamma', 'beta', 'LayerNorm']     # :422-427
    named = list(model.named_parameters())
    groups = [{'params': [p for n, p in named if not any(nd in n for nd in no_decay)], 'weight_decay': 0.01},
              {'params': [p for n, p in named if any(nd in n for nd in no_decay)], 'weight_decay': 0.0}]
    optimizer = FusedLAMBAMP(groups, lr=learning_rate)
    lr_scheduler = PolyWarmUpScheduler(optimizer, warmup=warmup_proportion, total_steps=max_steps,
                                       base_lr=learning_rate, device=device)
    grad_scaler = torch.amp.GradScaler("cuda", init_scale=init_loss_scale, enabled=use_grad_scaler)
    if distributed:
        from torch.nn.parallel import DistributedDataParallel as DDP
        side = torch.cuda.Stream()
        with torch.cuda.stream(side):
            model = DDP(model, device_ids=[device.index], output_device=device.index, bucket_cap_mb=bucket_cap_mb,
                        gradient_as_bucket_view=True)
        torch.cuda.current_stream().wait_stream(side)
    optimizer.setup_fp32_params()                          # :477 (after the DDP wrap, as in the reference)
    criterion = BertPretrainingCriterion(config.vocab_size, sequence_output_is_dense=sequence_output_is_dense)
    return model, optimizer, grad_scaler, lr_scheduler, criterion, config


def take_training_step(grad_scaler, model, criterion, batch, loss_acc=None):
    prediction_scores, seq_relationship_score = model(input_ids=batch['input_ids'], token_type_ids=batch['token_type_ids'],
                                                      attention_mask=batch['attention_mask'], masked_lm_labels=batch['labels'])
    loss = criterion(prediction_scores, seq_relationship_score, batch['labels'], batch['next_sentence_labels'])
    if loss_acc is not None:
        loss_acc.add_(loss.detach().float())
    grad_scaler.scale(loss).backward()
    return loss


def take_optimizer_step(lr_scheduler, optimizer, grad_scaler):
    lr_scheduler.step()
    grad_scaler.step(optimizer)
    grad_scaler.update()
    optimizer.zero_grad(set_to_none=True)


def capture_step_graph(fn, warmup_iters=11):
    """Capture `fn` (a whole training step or a gradient-accumulation micro-step) into a CUDA graph the way the reference driver
    does (run_pretraining.py:611-640): `warmup_iters` eager executions on a side stream first (lazy optimizer state, DDP bucket
    rebuild, cuBLAS/NCCL initialisation must all have happened -- the reference uses 11 for DDP), then one captured execution.
    Requirements the product path meets: static shapes (nonzero_static row gather), no host synchronisation, dropout masks keyed by
    the device step counter (ops.step_counter), LAMB tables patched by a capturable copy.  Returns the torch.cuda.CUDAGraph."""
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(warmup_iters):
            fn()
    torch.cuda.current_stream().wait_stream(side)
    # fp32 parameters: the graph must contain the bf16 casts it reads (ops.w16).  A copy the warm-ups cached is valid now, but a
    # replay that reused it would read the weights of capture time on every replay, however the optimizer changed them since.
    ops.weight_epoch["n"] += 1
    graph = torch.cuda.CUDAGraph()
    # thread_local: CUDA calls made by OTHER host threads during the capture (NCCL watchdog, data-loader pinning) must not invalidate it
    with torch.cuda.graph(graph, capture_error_mode="thread_local"):
        fn()
    return graph


# ------------------------------------------------------------------------------------------------------------------
# multi-GPU host logic (one process per GPU, pure data parallelism: run_pretraining.py:338,455-475,544-547)
# ------------------------------------------------------------------------------------------------------------------
def rank_seed(base_seed, rank):
    """Each rank draws its own micro-batches: seed + rank (run_pretraining.py:544-547 seeds with seed + local_rank)."""
    return int(base_seed) + int(rank)


def max_over_ranks(value_ms, device="cpu"):
    """A multi-GPU step takes as long as its slowest rank: MAX-reduce the device-timed milliseconds."""
    import torch.distributed as dist
    t = torch.tensor([float(value_ms)], device=device)
    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return t.item()


def global_throughput(micro_batch, world, steps, ms_total):
    """training_sequences_per_second exactly as the reference computes it (run_pretraining.py:748)."""
    return micro_batch * world * steps / (ms_total / 1000.0)
