"""Padding-free training throughput: BERT-large pretraining steps (forward, backward, LAMB) at B = 128, S = 512, dropout 0.1, 1xH100, on
a variable-length batch (lengths ~ U{128..512} rounded up to 64, the distribution of tools/bench_infer.py) with MLM labels on kept
positions only (80 per row).  The padded eager step and the padding-free eager step (BertModel.remove_padding(True, training=True):
packed tokens, variable-length attention forward and backward) alternate, three runs each; one padded CUDA-graph leg gives context
(the padding-free route reads the mask on the host every step, so it is not graph-capturable).  Each leg reports ms/step, sequences/s,
real tokens/s and peak memory.  Last, with every dropout off, the loss of both routes on the batch is compared bit for bit.
Writes bench_out/bench_train_packed.json."""
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from deeplearningexamples_b200 import ops, training as T  # noqa: E402


def gpu_info():
    """Name and power limit of the card the run is on (read-only nvidia-smi query, as in tools/bench_infer.py)."""
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


B, S, P = int(os.environ.get("B", 128)), int(os.environ.get("S", 512)), 80
cfg = dict(T.BERT_LARGE)
device = torch.device("cuda", 0)
model, opt, scaler, sched, crit, config = T.prepare_model_and_optimizer(cfg, device, seed=42, static_masked_count=B * P)

g = torch.Generator().manual_seed(1)
batch = T.synthetic_batch(B, S, config.vocab_size, P, seed=1, full_mask=True)
lens = ((torch.randint(S // 4, S + 1, (B,), generator=g) + 63) // 64 * 64).clamp(max=S)
am = (torch.arange(S).unsqueeze(0) < lens.unsqueeze(1)).to(torch.int64)
labels = torch.full((B, S), -1, dtype=torch.int64)
for b in range(B):                                      # the MLM positions among the kept ones
    pos = torch.randperm(int(lens[b]), generator=g)[:P]
    labels[b, pos] = torch.randint(0, 30522, (pos.numel(),), generator=g)
batch.update(attention_mask=am, labels=labels)
batch = {k: v.to(device) for k, v in batch.items()}
tokens = int(lens.sum())

out = dict(workload=f"BERT-large pretraining step seq{S} bs{B} dropout 0.1, variable-length batch", **gpu_info(),
           token_fill=round(tokens / (B * S), 3), runs=[])
print(json.dumps({k: v for k, v in out.items() if k != "runs"}), flush=True)


def one_step():
    T.take_training_step(scaler, model, crit, batch)
    T.take_optimizer_step(sched, opt, scaler)


def measure(padding_free, graphs, rep=None, n=8):
    model.remove_padding(padding_free, training=padding_free)
    run = one_step
    if graphs:
        run = T.capture_step_graph(one_step, warmup_iters=3).replay
    for _ in range(3):
        run()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        run()
    e1.record()
    torch.cuda.synchronize()
    model.remove_padding(False)
    ms = e0.elapsed_time(e1) / n
    r = dict(route="padding-free" if padding_free else "padded", cuda_graph=graphs, ms_per_step=round(ms, 2),
             sequences_per_s=round(B / ms * 1e3, 1), real_tokens_per_s=round(tokens / ms * 1e3),
             peak_memory_gib=round(torch.cuda.max_memory_allocated() / 2 ** 30, 2))
    if rep is not None:
        r["run"] = rep
    out["runs"].append(r)
    print(r, flush=True)


for rep in range(3):                                    # padded and padding-free eager legs alternate
    measure(False, False, rep)
    measure(True, False, rep)
measure(False, True)

# output check: every dropout off, the two routes' losses on the batch
for m in model.modules():
    if isinstance(m, torch.nn.Dropout):
        m.p = 0.0
losses = []
for padding_free in (False, True):
    model.remove_padding(padding_free, training=padding_free)
    ops.manual_seed(3)
    with torch.no_grad():
        scores, nsp = model(batch["input_ids"], batch["token_type_ids"], batch["attention_mask"], batch["labels"])
        losses.append(crit(scores, nsp, batch["labels"], batch["next_sentence_labels"]).float())
model.remove_padding(False)
out["dropout_off_loss"] = dict(padded=losses[0].item(), padding_free=losses[1].item(), bit_identical=bool(torch.equal(*losses)))
print(out["dropout_off_loss"], flush=True)
print(json.dumps(out))
os.makedirs("bench_out", exist_ok=True)
json.dump(out, open("bench_out/bench_train_packed.json", "w"))
