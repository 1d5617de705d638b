"""Packed SWAG fine-tuning throughput: BERT-large SWAG steps (BertForMultipleChoice, 4 choices; forward, backward, FusedAdam with
global-norm clip 1.0, device-side warmup_linear schedule) at dropout 0.1, 1xH100, on a synthetic stand-in for a SWAG example stream
(swag.synthetic_swag_features: contexts ~ U{S/16..S/4}, endings ~ U{S/32..S/8} tokens at choice length S = 128, no claim about the
real SWAG data).  Two CUDA-graph legs alternate, three runs each, on the same seeded example stream:

  padded   the padded step on E examples as [E, 4, 128] (4E choice rows; run_swag.sh pads every choice to 128);
  packed   the packed step on the same token capacity as rows of 512 (E*4*128/512 rows, k = 16: up to 4 whole examples per row),
           packed from the stream (packing.PackedLoader(swag=True)).

Each leg reports ms/step, examples/s, real tokens/s, token fill and peak memory (the padded leg also its model TFLOP/s).  Then an eval-mode forward pair, each captured into a
CUDA graph: examples/s of the padded and the packed forward.  --examples 12 is run_swag.sh's per-GPU batch.  Writes
<out>/bench_swag_packed.json."""
import argparse
import gc
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from deeplearningexamples_b200 import ops, packing, swag as W, training as T  # noqa: E402


def gpu_info():
    """Name, power limit and max SM clock of the card the run is on (a read-only nvidia-smi query)."""
    info = dict(gpu=torch.cuda.get_device_name())
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=pci.bus_id,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        bus = getattr(torch.cuda.get_device_properties(torch.cuda.current_device()), "pci_bus_id", None)
        rows = [r.split(", ") for r in q]
        mine = [r for r in rows if bus is not None and r[0].lower().endswith(str(bus).lower()[-7:])] or rows[:1]
        info.update(power_limit=mine[0][1], max_sm_clock=mine[0][2])
    except Exception as e:                                        # the numbers below still stand; the context is missing
        info.update(power_limit=f"unknown ({e})")
    return info


ap = argparse.ArgumentParser()
ap.add_argument("--steps", type=int, default=20)
ap.add_argument("--examples", type=int, default=32, help="examples per padded step (run_swag.sh: 12 per GPU)")
ap.add_argument("--choice_len", type=int, default=128, help="padded length of one choice row (run_swag.sh: max_seq_length 128)")
ap.add_argument("--seq", type=int, default=512, help="packed row length")
ap.add_argument("--per_row", type=int, default=16, help="sample slots per packed row, a multiple of the 4 choices")
ap.add_argument("--out", default="bench_out")
args = ap.parse_args()

C = 4
E, SC, S, KPR = args.examples, args.choice_len, args.seq, args.per_row
if (E * C * SC) % S != 0:
    raise SystemExit(f"--examples * 4 * --choice_len must be a multiple of --seq, got {E} * 4 * {SC} and {S}")
R = E * C * SC // S                                               # packed rows of the same token capacity
cfg = dict(T.BERT_LARGE)
device = torch.device("cuda", 0)
state = {}

source = [W.synthetic_swag_features(E, C, SC, cfg["vocab_size"], seed=1 + i) for i in range(48)]
# first-fit decreasing places the longest examples first, so the first batches of a stream hold fewer, longer examples: the packed
# leg times a batch from the middle of the stream, and the stream's averages over its full batches are reported next to it
stream = list(packing.PackedLoader(source, R, S, KPR, swag=True, num_choices=C))
packed_host = stream[len(stream) // 2]
full = stream[2:-2]
stream_stats = dict(packed_batches=len(stream), mean_examples_per_row=round(sum(b.num_samples for b in full) / (R * len(full)), 3),
                    mean_token_fill=round(sum(packing.token_fill(b) for b in full) / len(full), 3),
                    unpacked_token_fill=round(sum(packing.token_fill(b) for b in source) / len(source), 3))
legs = {"padded": ({k: v.to(device) for k, v in source[0].items()}, E, int(source[0]["input_mask"].sum())),
        "packed": ({k: v.to(device) for k, v in packed_host.items()}, packed_host.num_samples,
                   int((packed_host["input_mask"] != 0).sum()))}
FLOPS = W.swag_flops_per_example(cfg, SC, C)


def fresh_model(leg):
    """Every leg starts from the same weights and optimizer state."""
    state.clear()
    gc.collect()
    torch.cuda.empty_cache()
    ops.manual_seed(42)
    model, opt, sched = W.prepare_swag_model_and_optimizer(cfg, device, C, seed=42, total_steps=10000)
    model.pack_sequences(KPR if leg == "packed" else 0)
    state.update(model=model, opt=opt, sched=sched)
    return model, opt, sched


def timed(run):
    for _ in range(3):
        run()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.steps):
        run()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / args.steps


def measure(leg, rep):
    batch, examples, tokens = legs[leg]
    model, opt, sched = fresh_model(leg)
    model.train()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    loss_acc = torch.zeros((), device=device)
    graph = T.capture_step_graph(lambda: W.swag_training_step(model, opt, sched, batch, loss_acc), warmup_iters=3)
    ms = timed(graph.replay)
    r = dict(leg=leg, run=rep, cuda_graph=True, ms_per_step=round(ms, 2), examples_per_s=round(examples / ms * 1e3, 1),
             real_tokens_per_s=round(tokens / ms * 1e3), token_fill=round(tokens / (E * C * SC), 3), examples_per_step=examples,
             # the padded step's encoder FLOPs per second; a packed step does less work per example and has no comparable figure
             model_tflops=round(examples * FLOPS / ms * 1e-9, 1) if leg == "padded" else None,
             peak_memory_gib=round(torch.cuda.max_memory_allocated() / 2 ** 30, 2), loss_finite=bool(torch.isfinite(loss_acc).item()))
    del graph
    print(r, flush=True)
    return r


def measure_eval(leg, rep):
    batch, examples, _ = legs[leg]
    model, _, _ = fresh_model(leg)
    model.eval()
    args_ = (batch["input_ids"], batch["segment_ids"], batch["input_mask"])

    def fwd():
        with torch.no_grad():
            model(*args_)
    graph = T.capture_step_graph(fwd, warmup_iters=3)
    ms = timed(graph.replay)
    r = dict(leg=f"{leg} eval forward", run=rep, cuda_graph=True, ms_per_forward=round(ms, 2), examples_per_s=round(examples / ms * 1e3, 1))
    del graph
    print(r, flush=True)
    return r


out = dict(workload=f"BERT-large SWAG step, {C} choices, dropout 0.1, FusedAdam + clip 1.0; padded {E} x {C} x {SC}, packed {R} x {S} "
                    f"(k = {KPR}); synthetic examples, contexts U{{{max(1, SC // 16)}..{SC // 4}}}, endings "
                    f"U{{{max(1, SC // 32)}..{SC // 8}}} tokens",
           **gpu_info(), packing_stream=stream_stats, runs=[], eval=[])
print(json.dumps({k: v for k, v in out.items() if k not in ("runs", "eval")}), flush=True)
for rep in range(3):
    for leg in ("padded", "packed"):
        out["runs"].append(measure(leg, rep))
for rep in range(2):
    for leg in ("padded", "packed"):
        out["eval"].append(measure_eval(leg, rep))
ops.check_device_errors()
print(json.dumps(out))
os.makedirs(args.out, exist_ok=True)
json.dump(out, open(os.path.join(args.out, "bench_swag_packed.json"), "w"), indent=1)
