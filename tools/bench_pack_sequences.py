"""Sequence-packing training throughput: BERT-large pretraining steps (forward, backward, LAMB) at S = 512, dropout 0.1, 1xH100, on the
length distribution of tools/bench_train_packed.py (lengths ~ U{128..512} rounded up to 64), MLM labels on ~15 % of each sample's real
tokens.  Three legs alternate, three runs each:

  padded        the padded CUDA-graph step on B = 128 unpacked rows (one sample per row);
  padding-free  the padding-free eager step on the same rows (BertModel.remove_padding(True, training=True));
  packed        the packed CUDA-graph step on B = 128 rows packed from the same sample stream (packing.PackedLoader, k = 3).

Each leg reports ms/step, rows/s, samples/s, real tokens/s, token fill and peak memory.  Writes bench_out/bench_pack_sequences.json.

With --profile, one eager padded step and one eager packed step instead run under torch.profiler (CUDA activities), and the attention
kernels' device time of the packed step is compared with what the padded step's attention time predicts from the tiles the varlen
kernels walk (sum over sequences of ceil(len/64)^2 against B * (S/64)^2).  Writes bench_out/bench_pack_sequences_profile.json."""
import argparse
import gc
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from deeplearningexamples_b200 import kernels as K, ops, packing, training as T  # noqa: E402


def gpu_info():
    """Name and power limit of the card the run is on (read-only nvidia-smi query, as in tools/bench_train_packed.py)."""
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
ap.add_argument("--profile", action="store_true")
ap.add_argument("--steps", type=int, default=8)
args = ap.parse_args()

B, S, P, KPR = 128, 512, 80, 3
cfg = dict(T.BERT_LARGE)
device = torch.device("cuda", 0)
state = {}


def fresh_model():
    """Every leg starts from the same weights and optimizer state; a new optimizer also has a new LAMB plan, which takes a bounded
    number of captured table updates (one per captured step)."""
    state.clear()
    gc.collect()
    torch.cuda.empty_cache()
    ops.manual_seed(42)
    state["m"] = T.prepare_model_and_optimizer(cfg, device, seed=42, static_masked_count=B * P)


fresh_model()
source = [packing.synthetic_varlen_batch(B, S, state["m"][5].vocab_size, P, seed=1 + i, round_to=64) for i in range(16)]
unpacked = {k: v.to(device) for k, v in source[0].items()}
# first-fit decreasing places the longest samples first, so the first batches of a stream hold fewer, longer samples: the packed leg
# times a batch from the middle of the stream, and the stream's averages over its full batches are reported next to it
stream = list(packing.PackedLoader(source, B, S, KPR, P))
packed_host = stream[len(stream) // 2]
full = stream[2:-2]
stream_stats = dict(packed_batches=len(stream), mean_samples_per_row=round(sum(b.num_samples for b in full) / (B * len(full)), 3),
                    mean_token_fill=round(sum(packing.token_fill(b) for b in full) / len(full), 3))
packed = {k: v.to(device) for k, v in packed_host.items()}
legs = {"padded": (unpacked, B, int(source[0]["attention_mask"].sum())),
        "padding-free": (unpacked, B, int(source[0]["attention_mask"].sum())),
        "packed": (packed, packed_host.num_samples, int((packed_host["attention_mask"] != 0).sum()))}


def set_route(leg):
    model = state["m"][0]
    model.remove_padding(leg == "padding-free", training=leg == "padding-free")
    model.pack_sequences(KPR if leg == "packed" else 0)


def step(batch):
    model, opt, scaler, sched, crit, _ = state["m"]
    T.take_training_step(scaler, model, crit, batch)
    T.take_optimizer_step(sched, opt, scaler)


def measure(leg, rep):
    batch, samples, tokens = legs[leg]
    fresh_model()
    set_route(leg)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    graph = None
    run = lambda: step(batch)
    if leg != "padding-free":
        graph = T.capture_step_graph(run, warmup_iters=3)
        run = graph.replay
    for _ in range(3):
        run()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.steps):
        run()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / args.steps
    r = dict(leg=leg, run=rep, cuda_graph=graph is not None, ms_per_step=round(ms, 2), rows_per_s=round(B / ms * 1e3, 1),
             samples_per_s=round(samples / ms * 1e3, 1), real_tokens_per_s=round(tokens / ms * 1e3), token_fill=round(tokens / (B * S), 3),
             samples_per_step=samples, peak_memory_gib=round(torch.cuda.max_memory_allocated() / 2 ** 30, 2))
    del graph, run
    print(r, flush=True)
    return r


def profile():
    from torch.profiler import ProfilerActivity, profile as tprof
    res = {}
    for leg in ("padded", "packed"):
        batch = legs[leg][0]
        set_route(leg)
        for _ in range(2):
            step(batch)
        torch.cuda.synchronize()
        with tprof(activities=[ProfilerActivity.CUDA]) as prof:
            step(batch)
            torch.cuda.synchronize()
        kern = {}
        for e in prof.events():
            if e.device_type == torch.autograd.DeviceType.CUDA:
                kern[e.name] = kern.get(e.name, 0.0) + e.device_time_total / 1e3
        attn = {n: round(ms, 3) for n, ms in kern.items() if "attn_" in n}
        res[leg] = dict(device_busy_ms=round(sum(kern.values()), 2), attention_ms=round(sum(attn.values()), 2), attention_kernels=attn,
                        top=sorted(((round(ms, 2), n[:100]) for n, ms in kern.items()), reverse=True)[:15])
    cu, _, _ = K.segment_table(packed["attention_mask"], KPR)
    lens = torch.diff(cu.long()).cpu()
    tiles = int(((lens + 63) // 64).pow(2).sum())
    full = B * (S // 64) ** 2
    res["packed"].update(sequences=int(lens.numel()), empty_sequences=int((lens == 0).sum()), tiles_walked=tiles, tiles_padded=full,
                         sum_len_sq_over_padded=round(float(lens.double().pow(2).sum()) / (B * S * S), 4),
                         predicted_attention_ms=round(res["padded"]["attention_ms"] * tiles / full, 2))
    res["packed"]["attention_over_prediction"] = round(res["packed"]["attention_ms"] / res["packed"]["predicted_attention_ms"], 3)
    return res


out = dict(workload=f"BERT-large pretraining step seq{S} bs{B} dropout 0.1, LAMB; U{{128..512}}/64 lengths, 15 % MLM labels; k = {KPR}",
           **gpu_info(), packing_stream=stream_stats, runs=[])
print(json.dumps({k: v for k, v in out.items() if k != "runs"}), flush=True)
os.makedirs("bench_out", exist_ok=True)
if args.profile:
    out["profile"] = profile()
    print(json.dumps(out["profile"], indent=1))
    json.dump(out, open("bench_out/bench_pack_sequences_profile.json", "w"), indent=1)
else:
    for rep in range(3):
        for leg in ("padded", "padding-free", "packed"):
            out["runs"].append(measure(leg, rep))
    ops.check_device_errors()
    print(json.dumps(out))
    json.dump(out, open("bench_out/bench_pack_sequences.json", "w"), indent=1)
