"""Packed GLUE fine-tuning throughput: BERT-large GLUE steps (forward, backward, FusedAdam without clipping, device-side linear
schedule) at S = 128, dropout 0.1, 1xH100, on a synthetic stand-in for a sentence-pair stream (glue.synthetic_glue_features: lengths
~ U{S/8..S/2}, no claim about any real GLUE task).  Two CUDA-graph legs alternate, three runs each, on the same seeded example stream:

  padded   the padded step on B unpacked rows (one example per row);
  packed   the packed step on B rows packed from the stream (packing.PackedLoader(glue=True), k examples per row at most).

Each leg reports ms/step, samples/s, real tokens/s, token fill and peak memory.  Then an eval-mode forward pair, each captured into a
CUDA graph: samples/s of the padded and the packed forward on the same batches.  Writes <out>/bench_glue_packed.json."""
import argparse
import gc
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from deeplearningexamples_b200 import glue as G, ops, packing, training as T  # noqa: E402


def gpu_info():
    """Name and power limit of the card the run is on (a read-only nvidia-smi query)."""
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
ap.add_argument("--batch", type=int, default=32)
ap.add_argument("--seq", type=int, default=128)
ap.add_argument("--per_row", type=int, default=4)
ap.add_argument("--num_labels", type=int, default=3)
ap.add_argument("--out", default="bench_out")
args = ap.parse_args()

B, S, KPR, NL = args.batch, args.seq, args.per_row, args.num_labels
cfg = dict(T.BERT_LARGE)
device = torch.device("cuda", 0)
state = {}

source = [G.synthetic_glue_features(B, S, cfg["vocab_size"], NL, seed=1 + i) for i in range(16)]
# first-fit decreasing places the longest examples first, so the first batches of a stream hold fewer, longer examples: the packed
# leg times a batch from the middle of the stream, and the stream's averages over its full batches are reported next to it
stream = list(packing.PackedLoader(source, B, S, KPR, glue=True))
packed_host = stream[len(stream) // 2]
full = stream[2:-2]
stream_stats = dict(packed_batches=len(stream), mean_samples_per_row=round(sum(b.num_samples for b in full) / (B * len(full)), 3),
                    mean_token_fill=round(sum(packing.token_fill(b) for b in full) / len(full), 3),
                    unpacked_token_fill=round(sum(packing.token_fill(b) for b in source) / len(source), 3))
legs = {"padded": ({k: v.to(device) for k, v in source[0].items()}, B, int(source[0]["input_mask"].sum())),
        "packed": ({k: v.to(device) for k, v in packed_host.items()}, packed_host.num_samples,
                   int((packed_host["input_mask"] != 0).sum()))}


def fresh_model(leg):
    """Every leg starts from the same weights and optimizer state."""
    state.clear()
    gc.collect()
    torch.cuda.empty_cache()
    ops.manual_seed(42)
    model, opt, sched = G.prepare_glue_model_and_optimizer(cfg, device, NL, seed=42, total_steps=10000)
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
    batch, samples, tokens = legs[leg]
    model, opt, sched = fresh_model(leg)
    model.train()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    loss_acc = torch.zeros((), device=device)
    graph = T.capture_step_graph(lambda: G.glue_training_step(model, opt, sched, batch, loss_acc), warmup_iters=3)
    ms = timed(graph.replay)
    r = dict(leg=leg, run=rep, cuda_graph=True, ms_per_step=round(ms, 2), samples_per_s=round(samples / ms * 1e3, 1),
             real_tokens_per_s=round(tokens / ms * 1e3), token_fill=round(tokens / (B * S), 3), samples_per_step=samples,
             peak_memory_gib=round(torch.cuda.max_memory_allocated() / 2 ** 30, 2), loss_finite=bool(torch.isfinite(loss_acc).item()))
    del graph
    print(r, flush=True)
    return r


def measure_eval(leg, rep):
    batch, samples, _ = legs[leg]
    model, _, _ = fresh_model(leg)
    model.eval()
    args_ = (batch["input_ids"], batch["segment_ids"], batch["input_mask"])

    def fwd():
        with torch.no_grad():
            model(*args_)
    graph = T.capture_step_graph(fwd, warmup_iters=3)
    ms = timed(graph.replay)
    r = dict(leg=f"{leg} eval forward", run=rep, cuda_graph=True, ms_per_forward=round(ms, 2), samples_per_s=round(samples / ms * 1e3, 1))
    del graph
    print(r, flush=True)
    return r


out = dict(workload=f"BERT-large GLUE step seq{S} bs{B} dropout 0.1, FusedAdam (no clip), {NL} labels; synthetic sentence pairs "
                    f"U{{{max(5, S // 8)}..{S // 2}}} tokens; k = {KPR}",
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
json.dump(out, open(os.path.join(args.out, "bench_glue_packed.json"), "w"), indent=1)
