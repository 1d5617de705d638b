#!/usr/bin/env python
"""Time the UNMODIFIED reference training step on the GPU(s) of this box -- the denominator of the north_star's ">= 1.0x the
reference's own build" -- with exactly the harness bench.py uses for the H100 arm (CUDA events, max over ranks, barrier +
synchronize on both sides, W warm-up steps, K timed steps, resident and end-to-end passes).

    python tools/bench_reference_gpu.py --arm reference --batch 32 --steps 8 --warmup 3            # 1 GPU
    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port P \
        tools/bench_reference_gpu.py --arm reference --batch 32 ...                                  # N GPUs (DDP, NCCL)
    python tools/bench_reference_gpu.py --arm ours ...     # same harness, the reference's functions over shims/ours (drop-in path)

What runs (tools/run_reference_driver.py sets up the import path; nothing of the reference is edited):
    run_pretraining.parse_arguments / setup_training / prepare_model_and_optimizer / take_training_step / take_optimizer_step
    (PyTorch/LanguageModeling/BERT/run_pretraining.py:140-321,324-375,377-486,518-536) with the reference's headline flags
    --fp16 --allreduce_post_accumulation --allreduce_post_accumulation_fp16 (scripts/run_pretraining.sh: model.half(), fp16 gradients,
    fp32 masters in FusedLAMBAMP, single-bucket DDP), its modeling.py and its fused_lamb_CUDA kernels (oracle/_ref); --mode amp selects
    the other reference path (fp32 parameters + torch.cuda.amp.autocast).  The process is launched as a 1-rank distributed job when not
    under torchrun, exactly as the reference's launch script does, because the script only takes the model.half() path when
    local_rank != -1 (run_pretraining.py:328-332).
Prints ONE JSON line on rank 0.
"""
import argparse
import json
import os
import socket
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
_T0 = time.time()


def log(msg):
    print(f"[refbench +{time.time() - _T0:7.1f}s] {msg}", file=sys.stderr, flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--arm", default="reference", choices=["reference", "ours"])
    ap.add_argument("--mode", default="fp16", choices=["fp16", "amp"])
    ap.add_argument("--seq", type=int, default=512)
    ap.add_argument("--batch", type=int, default=32, help="per-GPU micro-batch (the reference's own: 32 @512, README.md:815)")
    ap.add_argument("--max-pred", type=int, default=0)
    ap.add_argument("--steps", type=int, default=8)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--jit", action="store_true", help="do NOT pass --disable_jit_fusions (torch.jit.script the model as the reference does by default)")
    ap.add_argument("--cuda-graphs", action="store_true", help="capture the step as the reference's --cuda_graphs does (run_pretraining.py:602-626)")
    ap.add_argument("--no-dropout", action="store_true")
    a = ap.parse_args()

    if "RANK" not in os.environ:                       # 1-rank distributed job (see module docstring)
        with socket.socket() as s:
            s.bind(("127.0.0.1", 0))
            port = s.getsockname()[1]
        os.environ.update(RANK="0", WORLD_SIZE="1", LOCAL_RANK="0", MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])

    import run_reference_driver as drv
    script = drv.setup(a.arm)
    import importlib.util
    import torch
    import torch.distributed as dist
    P = a.max_pred or (80 if a.seq >= 384 else 20)
    cfg_path = os.path.join(drv.REF, "bert_configs", "large.json")
    if a.no_dropout:
        cfg = json.load(open(cfg_path))
        cfg["hidden_dropout_prob"] = cfg["attention_probs_dropout_prob"] = 0.0
        cfg_path = os.path.join("/tmp", f"large_nodrop_{rank}.json")
        json.dump(cfg, open(cfg_path, "w"))
    out_dir = f"/tmp/refbench_{os.getpid()}"
    argv = [script, "--input_dir", f"synthetic?seq_len={a.seq}&max_pred={P}&samples={4 * a.batch * world}", "--config_file", cfg_path,
            "--output_dir", out_dir, "--vocab_file", "vocab.txt", "--train_batch_size", str(a.batch), "--max_seq_length", str(a.seq), "--max_predictions_per_seq", str(P),
            "--max_steps", "7038", "--warmup_proportion", "0.128", "--learning_rate", "4e-3", "--seed", "42", "--do_train", "--skip_checkpoint",
            "--json-summary", os.path.join(out_dir, "dllogger.json"), "--fp16"]
    if a.mode == "fp16":
        argv += ["--allreduce_post_accumulation", "--allreduce_post_accumulation_fp16"]
    if not a.jit:
        argv += ["--disable_jit_fusions"]
    if a.cuda_graphs:
        # the reference's graph mode only captures with --no_dense_sequence_output: its dense path calls torch.nonzero (modeling.py:590)
        # and its criterion indexes labels with a boolean mask (run_pretraining.py:89), both of which synchronise
        argv += ["--cuda_graphs", "--no_dense_sequence_output"]
    sys.argv = argv
    spec = importlib.util.spec_from_file_location("run_pretraining", script)
    rp = importlib.util.module_from_spec(spec)
    sys.modules["run_pretraining"] = rp
    spec.loader.exec_module(rp)                       # the unmodified reference driver, imported as a module (its main() is not called)

    args = rp.parse_arguments()
    device, args = rp.setup_training(args)
    model, optimizer, grad_scaler, lr_scheduler, checkpoint, global_step, criterion, epoch = rp.prepare_model_and_optimizer(
        args, device, sequence_output_is_dense=not args.no_dense_sequence_output)
    model.train()
    stats = rp.SyncFreeStats()                         # as main() does (:584-597)
    stats.add_stat('model_step')
    stats.add_stat('optimizer_step', dtype=torch.int32, device_func=(lambda: optimizer.param_groups[0]['step']))
    stats.add_stat('average_loss', dtype=torch.float32, device_tensor=torch.zeros(1, dtype=torch.float32, device=device))
    stats.add_stat('learning_rate', dtype=torch.float32, device_func=(lambda: optimizer.param_groups[0]['lr']))

    from deeplearningexamples_b200 import training as T          # synthetic batch generator + throughput formula only
    host = [T.synthetic_batch(a.batch, a.seq, 30528, P, seed=T.rank_seed(42, rank) + 100 * i, pin=True) for i in range(4)]
    dev = [{k: v.to(device) for k, v in hb.items()} for hb in host[:2]]
    stage = {k: torch.empty_like(v, device=device) for k, v in host[0].items()}
    loss_host = torch.zeros(1, dtype=torch.float32).pin_memory()
    h2d = sum(v.numel() * v.element_size() for v in host[0].values())
    graph = {"g": None}

    def one_step():
        rp.take_training_step(args, grad_scaler, model, criterion, stage, stats)
        rp.take_optimizer_step(args, lr_scheduler, optimizer, grad_scaler, device, stats)

    def run_step():
        graph["g"].replay() if graph["g"] is not None else one_step()

    def step_resident(i):
        for k in stage:
            stage[k].copy_(dev[i % 2][k], non_blocking=True)
        run_step()

    def step_e2e(i):
        for k in stage:
            stage[k].copy_(host[i % 4][k], non_blocking=True)
        run_step()
        loss_host.copy_(stats.device_stat('average_loss'), non_blocking=True)

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    def timed(fn, steps):
        barrier()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        t = time.perf_counter()
        for i in range(steps):
            fn(i)
        e1.record()
        t = time.perf_counter() - t
        barrier()
        log(f"  host enqueue {1000 * t / steps:.2f} ms/step vs device {e0.elapsed_time(e1) / steps:.2f} ms/step")
        return T.max_over_ranks(e0.elapsed_time(e1), device)

    log(f"arm={a.arm} mode={a.mode} B={a.batch} S={a.seq} world={world} jit={a.jit} graphs={a.cuda_graphs}")
    n_warm = max(a.warmup, 3)
    for k in stage:
        stage[k].copy_(dev[0][k])
    if a.cuda_graphs:
        n_warm = max(n_warm, 11)
        graph["g"] = T.capture_step_graph(one_step, warmup_iters=n_warm)      # same sequence as run_pretraining.py:611-626
    else:
        for i in range(n_warm):
            step_resident(i)
    step_e2e(0)
    torch.cuda.synchronize()
    log("warm-up done")
    ms_res = timed(step_resident, a.steps)
    ms_e2e = timed(step_e2e, a.steps)
    value = T.global_throughput(a.batch, world, a.steps, ms_res)
    e2e = T.global_throughput(a.batch, world, a.steps, ms_e2e)
    line = {"impl": "reference_gpu" if a.arm == "reference" else "ours_via_reference_driver", "metric": "training_sequences_per_second",
            "value": round(value, 2), "unit": "sequences/s", "n_gpus": world, "steps": a.steps, "warmup": n_warm,
            "ms_per_step": round(ms_res / a.steps, 3), "higher_is_better": True, "scaling": "weak",
            "dtype": ("fp16" if a.arm == "reference" else "bf16") + (" parameters (model.half())" if a.mode == "fp16" else " autocast over fp32 parameters"),
            "data": "synthetic",
            "e2e": {"value": round(e2e, 2), "unit": "sequences/s", "h2d_bytes_per_step": h2d, "d2h_bytes_per_step": 4, "ms_per_step": round(ms_e2e / a.steps, 3)},
            "config": {"workload": f"BERT-large pretraining step seq{a.seq} LAMB, reference run_pretraining.py functions", "seq_len": a.seq,
                       "micro_batch_per_gpu": a.batch, "global_batch": a.batch * world, "max_predictions_per_seq": P,
                       "dropout": 0.0 if a.no_dropout else 0.1, "parallelism": f"dp{world}", "cuda_graphs": a.cuda_graphs,
                       "torchscript": a.jit, "flags": " ".join(argv[1:])},
            "hbm_peak_gb": round(torch.cuda.max_memory_allocated() / 2 ** 30, 1), "final_loss_acc": round(loss_host.item(), 4)}
    if rank == 0:
        print(json.dumps(line), flush=True)
    if dist.is_initialized():
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
