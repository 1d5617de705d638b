"""BERT pretraining driver with the reference's argument, checkpoint and metric surface.

Mirror of PyTorch/LanguageModeling/BERT/run_pretraining.py (NVIDIA/DeepLearningExamples): every flag of
parse_arguments (:140-321) is accepted; checkpoints are `ckpt_{step}.pt` = {'model','optimizer','grad_scaler','epoch'}
(:494-504) and resume follows :388-410,440-449 (phase-2 offset, step/lr reset on phase change, newest-3 retention);
the reported metric is training_sequences_per_second = batch * world * (steps - skipped) / seconds (:748).

What is different, and why:
  * 16-bit training is bf16 (`--fp16` / `--amp` select it); with `--allreduce_post_accumulation_fp16` the model itself is cast
    (`model.bfloat16()`, the reference's `model.half()`), otherwise parameters stay fp32 and the kernels run on bf16 copies.
  * `lddl`, `dllogger`, `h5py`, `apex` are not importable offline: batches come from `SyntheticPretrainLoader` (the lddl batch
    format: five int64 tensors) unless a real `lddl` is installed and `--input_dir` exists; logging is a JSON-lines shim.
  * TorchScript is not applicable to custom autograd functions: `--disable_jit_fusions` is implied.
  * `--cuda_graphs` captures the whole step (and the gradient-accumulation micro-step) exactly as the reference does (:602-640,669);
    dropout stays on: masks are keyed by a device-side step counter (ops.step_counter) that the captured forward bumps.
  * `--remove_padding` (not in the reference) trains padding-free: every encoder layer runs on the real tokens of the batch only
    (BertModel.remove_padding(True, training=True)).  It reads each batch's mask on the host, so it excludes `--cuda_graphs`, and it
    excludes `--checkpoint_activations`.
  * `--pack_sequences K` (not in the reference) packs up to K samples into each row (packing.PackedLoader over the loader, and
    BertPreTrainedModel.pack_sequences(K)).  Shapes stay static, so it works with `--cuda_graphs`, gradient accumulation and DDP; it
    excludes `--remove_padding` and `--checkpoint_activations`.  With `--input_dir synthetic` the samples have variable lengths.
    `training_sequences_per_second` still counts rows; `training_samples_per_second` counts the samples of the timed steps.
"""
import argparse
import json
import math
import os
import random
import signal
import time

import numpy as np
import torch
import torch.distributed as dist

from . import modeling, ops, packing
from .lamb import FusedLAMBAMP
from .schedulers import PolyWarmUpScheduler
from .training import BertPretrainingCriterion, capture_step_graph, synthetic_batch

timeout_sent = False


def _on_sigterm(sig, frame):          # cluster time-up: checkpoint at the next optimizer step and leave (:62-72)
    global timeout_sent
    timeout_sent = True


# ---------------------------------------------------------------------------------------------------------------------
# small stand-ins for the absent third-party modules
# ---------------------------------------------------------------------------------------------------------------------
class JsonLogger:
    """dllogger stand-in: one JSON object per line on rank 0 (same keys the reference logs)."""

    def __init__(self, path, enabled):
        self.enabled = enabled
        self.f = None
        if enabled and path:
            os.makedirs(os.path.dirname(os.path.abspath(path)) or ".", exist_ok=True)
            self.f = open(path, "a")

    def log(self, step, data):
        if not self.enabled:
            return
        rec = {"step": step if isinstance(step, str) else list(step), "data": data, "time": time.time()}
        line = json.dumps(rec, default=str)
        print("DLLL " + line, flush=True)
        if self.f:
            self.f.write(line + "\n")

    def flush(self):
        if self.f:
            self.f.flush()


class SyntheticPretrainLoader:
    """`lddl.torch.get_bert_pretrain_data_loader` stand-in: an iterable of pinned batches in the lddl format
    (input_ids, token_type_ids, attention_mask, labels, next_sentence_labels; int64; labels == -1 ignored), sharded by rank."""

    def __init__(self, batch_size, seq_len, max_pred, vocab, steps_per_epoch, base_seed, rank, n_distinct=8, variable_length=False):
        """variable_length: right-padded samples of U{S/4..S} tokens with MLM labels on ~15 % of them (packing.synthetic_varlen_batch)
        instead of full rows."""
        make = packing.synthetic_varlen_batch if variable_length else synthetic_batch
        self.batches = [make(batch_size, seq_len, vocab, max_pred, seed=base_seed + rank + 1000 * i, pin=torch.cuda.is_available())
                        for i in range(n_distinct)]
        self.steps_per_epoch = steps_per_epoch

    def __len__(self):
        return self.steps_per_epoch

    def __iter__(self):
        for i in range(self.steps_per_epoch):
            yield self.batches[i % len(self.batches)]


# ---------------------------------------------------------------------------------------------------------------------
def parse_arguments(argv=None):
    p = argparse.ArgumentParser(description="BERT pretraining (H100-native kernels, reference argument surface)")
    p.add_argument("--input_dir", default=None, type=str, help="LDDL shards directory, or 'synthetic' (default when lddl is absent)")
    p.add_argument("--config_file", default=None, type=str, required=True, help="BERT config json (bert_configs/large.json)")
    p.add_argument("--output_dir", default=None, type=str, required=True)
    p.add_argument("--vocab_file", type=str, default=None)
    p.add_argument("--init_checkpoint", default=None, type=str)
    p.add_argument("--max_seq_length", default=512, type=int)
    p.add_argument("--max_predictions_per_seq", default=80, type=int)
    p.add_argument("--train_batch_size", default=32, type=int)
    p.add_argument("--learning_rate", default=5e-5, type=float)
    p.add_argument("--num_train_epochs", default=3.0, type=float)
    p.add_argument("--max_steps", default=1000, type=float)
    p.add_argument("--warmup_proportion", default=0.01, type=float)
    p.add_argument("--local_rank", type=int, default=os.getenv('LOCAL_RANK', -1))
    p.add_argument("--seed", type=int, default=42)
    p.add_argument("--gradient_accumulation_steps", type=int, default=1)
    p.add_argument("--fp16", default=False, action="store_true", help="16-bit training (bf16 on H100)")
    p.add_argument("--amp", default=False, action="store_true", help="alias of --fp16")
    p.add_argument("--loss_scale", type=float, default=0.0)
    p.add_argument("--log_freq", type=float, default=1.0)
    p.add_argument("--checkpoint_activations", default=False, action="store_true")
    p.add_argument("--resume_from_checkpoint", default=False, action="store_true")
    p.add_argument("--resume_step", type=int, default=-1)
    p.add_argument("--num_steps_per_checkpoint", type=int, default=100)
    p.add_argument("--skip_checkpoint", default=False, action="store_true")
    p.add_argument("--phase2", default=False, action="store_true")
    p.add_argument("--resume_phase2", default=False, action="store_true")
    p.add_argument("--allreduce_post_accumulation", default=False, action="store_true")
    p.add_argument("--allreduce_post_accumulation_fp16", default=False, action="store_true")
    p.add_argument("--phase1_end_step", type=int, default=7038)
    p.add_argument("--init_loss_scale", type=int, default=2 ** 20)
    p.add_argument("--do_train", default=False, action="store_true")
    p.add_argument("--json-summary", type=str, default="results/dllogger.json", dest="json_summary")
    p.add_argument("--use_env", action="store_true")
    p.add_argument("--disable_progress_bar", default=False, action="store_true")
    p.add_argument("--steps_this_run", type=int, default=-1)
    p.add_argument("--profile", default=False, action="store_true")
    p.add_argument("--profile-start", type=int, default=0, dest="profile_start")
    p.add_argument("--num_workers", type=int, default=4)
    p.add_argument("--no_dense_sequence_output", default=False, action="store_true")
    p.add_argument("--disable_jit_fusions", default=False, action="store_true")
    p.add_argument("--cuda_graphs", default=False, action="store_true")
    p.add_argument("--remove_padding", default=False, action="store_true",
                   help="padding-free training: run the encoder on the real tokens of each batch only (BertModel.remove_padding)")
    p.add_argument("--pack_sequences", type=int, default=0, metavar="K",
                   help="pack up to K samples into each row (sequence packing, BertPreTrainedModel.pack_sequences); 0 = off")
    args = p.parse_args(argv)
    if args.remove_padding and (args.cuda_graphs or args.checkpoint_activations):
        raise ValueError("--remove_padding reads each batch's attention mask on the host: it cannot be combined with --cuda_graphs, "
                         "and the padding-free encoder does not support --checkpoint_activations")
    if args.pack_sequences < 0:
        raise ValueError("--pack_sequences takes K >= 1 samples per row (0 = off)")
    if args.pack_sequences and (args.remove_padding or args.checkpoint_activations):
        raise ValueError("--pack_sequences cannot be combined with --remove_padding (another route), and packed rows do not support "
                         "--checkpoint_activations")
    args.fp16 = args.fp16 or args.amp
    args.local_rank = int(args.local_rank)
    if args.steps_this_run < 0:
        args.steps_this_run = args.max_steps
    return args


def is_main_process():
    return (not dist.is_initialized()) or dist.get_rank() == 0


def get_world_size():
    return dist.get_world_size() if dist.is_initialized() else 1


def setup_training(args):
    if not torch.cuda.is_available():
        raise RuntimeError("run_pretraining needs a CUDA device: the H100 hot path has no CPU fallback")
    if args.local_rank == -1:
        device = torch.device("cuda", 0)
        args.allreduce_post_accumulation = False
        args.allreduce_post_accumulation_fp16 = False
    else:
        torch.cuda.set_device(args.local_rank)
        device = torch.device("cuda", args.local_rank)
        dist.init_process_group(backend='nccl', init_method='env://')
    args.n_gpu = 1
    if args.gradient_accumulation_steps < 1:
        raise ValueError("Invalid gradient_accumulation_steps parameter: {}, should be >= 1".format(args.gradient_accumulation_steps))
    if args.train_batch_size % args.gradient_accumulation_steps != 0:
        raise ValueError("Invalid gradient_accumulation_steps parameter: {}, batch size {} should be divisible".format(
            args.gradient_accumulation_steps, args.train_batch_size))
    args.train_batch_size = args.train_batch_size // args.gradient_accumulation_steps
    if not args.do_train:
        raise ValueError(" `do_train`  must be True.")
    if not args.resume_from_checkpoint and os.path.exists(args.output_dir) and any(f.startswith('ckpt') for f in os.listdir(args.output_dir)):
        raise ValueError("Output directory ({}) already exists and is not empty.".format(args.output_dir))
    if (not args.resume_from_checkpoint or not os.path.exists(args.output_dir)) and is_main_process():
        os.makedirs(args.output_dir, exist_ok=True)
    if args.cuda_graphs and args.no_dense_sequence_output is False and args.max_predictions_per_seq <= 0:
        raise ValueError("--cuda_graphs needs --max_predictions_per_seq > 0 (static number of gathered MLM rows)")
    return device, args


def prepare_model_and_optimizer(args, device, sequence_output_is_dense):
    config = modeling.BertConfig.from_json_file(args.config_file)
    if config.vocab_size % 8 != 0:
        config.vocab_size += 8 - (config.vocab_size % 8)
    model = modeling.BertForPreTraining(config, sequence_output_is_dense=sequence_output_is_dense)
    if sequence_output_is_dense:      # max_predictions_per_seq bounds the masked positions per sequence by definition of the data
        model.cls.static_masked_count = (args.train_batch_size) * args.max_predictions_per_seq
    checkpoint, global_step = None, 0
    if args.resume_from_checkpoint:
        if args.resume_step == -1 and not args.init_checkpoint:
            names = [f for f in os.listdir(args.output_dir) if f.endswith(".pt")]
            args.resume_step = max(int(x.split('.pt')[0].split('_')[1].strip()) for x in names)
        global_step = args.resume_step if not args.init_checkpoint else 0
        path = args.init_checkpoint or os.path.join(args.output_dir, "ckpt_{}.pt".format(global_step))
        checkpoint = torch.load(path, map_location=device, weights_only=False)
        model.load_state_dict(checkpoint['model'], strict=False)
        if args.phase2 and not args.init_checkpoint:
            global_step -= args.phase1_end_step
        if args.init_checkpoint:
            args.resume_step = 0
        if is_main_process():
            print("resume step from ", args.resume_step)
    model.to(device)
    if args.fp16 and args.allreduce_post_accumulation_fp16:
        model.bfloat16()
    no_decay = ['bias', 'gamma', 'beta', 'LayerNorm']
    named = list(model.named_parameters())
    groups = [{'params': [p for n, p in named if not any(nd in n for nd in no_decay)], 'weight_decay': 0.01},
              {'params': [p for n, p in named if any(nd in n for nd in no_decay)], 'weight_decay': 0.0}]
    optimizer = FusedLAMBAMP(groups, lr=args.learning_rate)
    lr_scheduler = PolyWarmUpScheduler(optimizer, warmup=args.warmup_proportion, total_steps=args.max_steps,
                                       base_lr=args.learning_rate, device=device)
    grad_scaler = torch.amp.GradScaler("cuda", init_scale=args.init_loss_scale, enabled=args.fp16)
    model.checkpoint_activations(args.checkpoint_activations)
    if args.remove_padding:
        model.remove_padding(True, training=True)
    if args.pack_sequences:
        model.pack_sequences(args.pack_sequences)
    if args.resume_from_checkpoint:
        if (args.phase2 and not args.resume_phase2) or args.init_checkpoint:
            for group in checkpoint['optimizer']['param_groups']:       # new phase: restart the schedule
                group['step'].zero_()
                group['lr'].fill_(args.learning_rate)
        elif 'grad_scaler' in checkpoint and (not args.phase2 or args.resume_phase2):
            grad_scaler.load_state_dict(checkpoint['grad_scaler'])
        optimizer.load_state_dict(checkpoint['optimizer'])
    if args.local_rank != -1:
        from torch.nn.parallel import DistributedDataParallel as DDP
        side = torch.cuda.Stream()
        with torch.cuda.stream(side):
            model = DDP(model, device_ids=[args.local_rank], output_device=args.local_rank, bucket_cap_mb=100,
                        gradient_as_bucket_view=True)
        torch.cuda.current_stream().wait_stream(side)
        if args.gradient_accumulation_steps > 1:
            from torch.distributed.algorithms.ddp_comm_hooks.default_hooks import allreduce_hook

            def hook(state, bucket):           # pre-divide by the accumulation steps, then the default allreduce (:460-475)
                bucket.set_buffer(bucket.buffer().div_(args.gradient_accumulation_steps))
                return allreduce_hook(state, bucket)
            model.register_comm_hook(None, hook)
    optimizer.setup_fp32_params()
    criterion = BertPretrainingCriterion(config.vocab_size, sequence_output_is_dense=sequence_output_is_dense)
    if (args.resume_from_checkpoint and not args.phase2) or args.resume_phase2 or args.init_checkpoint:
        start_epoch = checkpoint.get('epoch', 0)
    else:
        start_epoch = 0
    return model, optimizer, grad_scaler, lr_scheduler, checkpoint, global_step, criterion, start_epoch, config


def checkpoint_step(args, epoch, global_step, model, optimizer, grad_scaler, last3, logger):
    torch.cuda.synchronize()
    if not is_main_process() or args.skip_checkpoint:
        return
    logger.log("PARAMETER", {"checkpoint_step": global_step})
    to_save = model.module if hasattr(model, 'module') else model
    step_name = global_step if (args.resume_step < 0 or not args.phase2) else global_step + args.phase1_end_step
    path = os.path.join(args.output_dir, "ckpt_{}.pt".format(step_name))
    torch.save({'model': to_save.state_dict(), 'optimizer': optimizer.state_dict(), 'grad_scaler': grad_scaler.state_dict(),
                'epoch': epoch}, path)
    if path in last3:
        last3.remove(path)
    last3.append(path)
    if len(last3) > 3:
        os.remove(last3.pop(0))


def take_training_step(args, grad_scaler, model, criterion, batch, loss_acc):
    scores, nsp = model(input_ids=batch['input_ids'], token_type_ids=batch['token_type_ids'], attention_mask=batch['attention_mask'],
                        masked_lm_labels=batch['labels'])
    loss = criterion(scores, nsp, batch['labels'], batch['next_sentence_labels'])
    loss_acc.add_(loss.detach().float())
    grad_scaler.scale(loss).backward()


def take_optimizer_step(args, lr_scheduler, optimizer, grad_scaler, skipped_acc):
    lr_scheduler.step()
    grad_scaler.step(optimizer)
    if grad_scaler.is_enabled():
        skipped_acc.add_(optimizer._found_inf)               # before update() resets the inf tracker (:530-533)
    grad_scaler.update()
    # Captured graphs freeze "assign" vs "accumulate" for every gradient: with gradient accumulation under --cuda_graphs the gradient
    # buffers therefore stay allocated and are zeroed in place, so the micro-step graph and the full-step graph both ACCUMULATE into the
    # same static buffers (the reference's set_to_none=True, :536, is kept otherwise).
    optimizer.zero_grad(set_to_none=not (args.cuda_graphs and args.gradient_accumulation_steps > 1))


def capture_training_graphs(args, model, optimizer, grad_scaler, lr_scheduler, criterion, static_batch, loss_acc, skipped_acc):
    """reference :602-640: eager warm-up on a side stream, then one captured graph for the full step (micro-step + optimizer step) and,
    with gradient accumulation, one for the micro-step alone (no_sync under DDP).  Both read `static_batch`, which must hold a real
    batch (all-ones labels, as the reference uses, would mark every position as masked and trip the static masked-row bound), and add
    into `loss_acc` / `skipped_acc`.  The warm-ups train on the static batch, as the reference's do.  Returns (full_graph, accum_graph);
    accum_graph is None without gradient accumulation."""
    full_graph = capture_step_graph(lambda: (take_training_step(args, grad_scaler, model, criterion, static_batch, loss_acc),
                                             take_optimizer_step(args, lr_scheduler, optimizer, grad_scaler, skipped_acc)), warmup_iters=11)
    accum_graph = None
    if args.gradient_accumulation_steps > 1:
        def micro():
            if hasattr(model, "no_sync"):
                with model.no_sync():
                    take_training_step(args, grad_scaler, model, criterion, static_batch, loss_acc)
            else:
                take_training_step(args, grad_scaler, model, criterion, static_batch, loss_acc)
        accum_graph = capture_step_graph(micro, warmup_iters=3)
        optimizer.zero_grad(set_to_none=False)       # the warm-up / captured micro-steps accumulated into the static gradient buffers
    return full_graph, accum_graph


def main(argv=None):
    global timeout_sent
    signal.signal(signal.SIGTERM, _on_sigterm)
    args = parse_arguments(argv)
    rank_off = max(args.local_rank, 0)
    random.seed(args.seed + rank_off)
    np.random.seed(args.seed + rank_off)
    torch.manual_seed(args.seed + rank_off)
    ops.manual_seed(args.seed + rank_off)
    device, args = setup_training(args)
    logger = JsonLogger(args.json_summary, is_main_process())
    logger.log("PARAMETER", {"Config": [str(vars(args))]})
    model, optimizer, grad_scaler, lr_scheduler, checkpoint, global_resume_step, criterion, epoch, config = \
        prepare_model_and_optimizer(args, device, sequence_output_is_dense=not args.no_dense_sequence_output)

    loader = None
    if args.input_dir and args.input_dir != "synthetic" and os.path.isdir(args.input_dir):
        try:
            import lddl.torch
            loader = lddl.torch.get_bert_pretrain_data_loader(
                args.input_dir, local_rank=rank_off, vocab_file=args.vocab_file,
                data_loader_kwargs={'batch_size': args.train_batch_size * args.n_gpu, 'num_workers': args.num_workers, 'pin_memory': True},
                base_seed=args.seed, log_dir=os.path.join(args.output_dir, 'lddl_log'), start_epoch=epoch)
        except ImportError:
            loader = None
    if loader is None:
        steps_needed = int(args.steps_this_run * args.gradient_accumulation_steps) + 64
        loader = SyntheticPretrainLoader(args.train_batch_size, args.max_seq_length, args.max_predictions_per_seq, config.vocab_size,
                                         steps_needed, args.seed, dist.get_rank() if dist.is_initialized() else 0,
                                         variable_length=bool(args.pack_sequences))
    if args.pack_sequences:
        loader = packing.PackedLoader(loader, args.train_batch_size, args.max_seq_length, args.pack_sequences, args.max_predictions_per_seq,
                                      pin=True)
    logger.log("PARAMETER", {"SEED": args.seed, "train_start": True, "batch_size_per_gpu": args.train_batch_size,
                             "learning_rate": args.learning_rate})
    model.train()
    last3 = []
    loss_acc = torch.zeros(1, dtype=torch.float32, device=device)
    skipped_acc = torch.zeros(1, dtype=torch.float32, device=device)
    host = {k: torch.zeros(1, dtype=torch.float32).pin_memory() for k in ("loss", "lr", "skipped")}
    model_step, raw_train_start = 0, None
    timed_samples = 0               # samples of the timed steps, counted on the host (a packed batch reports its count)
    skip_for_perf = 50 if args.phase2 else 4
    static_batch = full_graph = accum_graph = None
    if args.cuda_graphs:
        first = next(iter(loader))
        static_batch = {k: v.to(device) for k, v in first.items()}
        full_graph, accum_graph = capture_training_graphs(args, model, optimizer, grad_scaler, lr_scheduler, criterion, static_batch,
                                                          loss_acc, skipped_acc)
        # the warm-up / capture executions advanced the optimizer: rewind the statistics the run reports (weights keep the 12+ steps,
        # exactly as in the reference, whose warm-up also trains on the static batch)
        loss_acc.zero_()
        skipped_acc.zero_()
    while True:
        for step, batch in enumerate(loader):
            model_step += 1
            accumulating = (model_step % args.gradient_accumulation_steps) != 0
            if raw_train_start is None and step == skip_for_perf:
                torch.cuda.synchronize()
                raw_train_start = time.time()
            if raw_train_start is not None:
                timed_samples += getattr(batch, "num_samples", args.train_batch_size)
            if args.cuda_graphs:
                for k in batch.keys():
                    static_batch[k].copy_(batch[k], non_blocking=True)
                (accum_graph if (accumulating and accum_graph is not None) else full_graph).replay()
            else:
                batch = {k: v.to(device, non_blocking=True) for k, v in batch.items()}
                if args.allreduce_post_accumulation and accumulating and hasattr(model, "no_sync"):
                    with model.no_sync():
                        take_training_step(args, grad_scaler, model, criterion, batch, loss_acc)
                else:
                    take_training_step(args, grad_scaler, model, criterion, batch, loss_acc)
                if not accumulating:
                    take_optimizer_step(args, lr_scheduler, optimizer, grad_scaler, skipped_acc)
            if not accumulating:
                host["loss"].copy_(loss_acc, non_blocking=True)
                host["lr"].copy_(optimizer.param_groups[0]['lr'].reshape(1), non_blocking=True)
                host["skipped"].copy_(skipped_acc, non_blocking=True)
            if (not accumulating) or timeout_sent:
                static_step = model_step // args.gradient_accumulation_steps
                dynamic_step = static_step - int(host["skipped"].item()) + global_resume_step
                no_log = static_step % args.log_freq
                if static_step + global_resume_step >= args.steps_this_run or timeout_sent:
                    torch.cuda.synchronize()
                    dynamic_step = static_step - int(skipped_acc.item()) + global_resume_step
                    if dynamic_step >= args.steps_this_run or timeout_sent:
                        train_time_raw = time.time() - (raw_train_start or time.time())
                        n_last = args.log_freq if no_log == 0 else no_log
                        loss_acc.div_(n_last * args.gradient_accumulation_steps)
                        if dist.is_initialized():
                            loss_acc.div_(get_world_size())
                            dist.all_reduce(loss_acc)
                        final_loss = loss_acc.item()
                        samples = torch.tensor([float(timed_samples)], device=device)
                        if dist.is_initialized():
                            dist.all_reduce(samples)
                        args.timed_samples = samples.item()
                        ops.check_device_errors()
                        (model.module if hasattr(model, "module") else model).cls.check_mlm_overflow()
                        logger.log((epoch, dynamic_step), {"final_loss": final_loss})
                        checkpoint_step(args, epoch, dynamic_step, model, optimizer, grad_scaler, last3, logger)
                        return args, train_time_raw, model_step, skip_for_perf, final_loss, logger
                if no_log == 0:
                    logger.log((epoch, dynamic_step), {"average_loss": host["loss"].item() / (args.log_freq * args.gradient_accumulation_steps),
                                                       "learning_rate": host["lr"].item(), "skipped_steps": int(host["skipped"].item())})
                    loss_acc.zero_()
                    if not args.skip_checkpoint and dynamic_step % args.num_steps_per_checkpoint == 0:
                        checkpoint_step(args, epoch, dynamic_step, model, optimizer, grad_scaler, last3, logger)
        epoch += 1


def cli(argv=None):
    t0 = time.time()
    args, train_time_raw, model_step, skip, final_loss, logger = main(argv)
    if is_main_process():
        perf = args.train_batch_size * get_world_size() * max(model_step - skip, 0) / max(train_time_raw, 1e-9)
        logger.log((), {"e2e_train_time": time.time() - t0, "training_sequences_per_second": perf,
                        "training_samples_per_second": args.timed_samples / max(train_time_raw, 1e-9), "final_loss": final_loss,
                        "raw_train_time": train_time_raw})
    logger.flush()
    if dist.is_initialized():
        dist.destroy_process_group()


if __name__ == "__main__":
    cli()
