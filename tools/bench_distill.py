"""General distillation throughput on one H100: the backbone step of distillation/general_distill.py (teacher BERT-base, student
6L-768D, distillation_config_backbone.json: attention-score KL + value-relation KL + hidden-state cosine, last-layer mapping, dropout 0.1,
FusedAdam with clip 1.0, device-side linear warm-up), B = 32, random token ids, full-length rows, the whole step as a CUDA graph.

Two legs per phase (S = 128 and S = 512), on the same models and batch:

  fused         the step as built: the relation-KL kernels on the layers' qkv / attention outputs (no [B, A, S, S] tensor)
  materialised  the same step with the two KL losses computed as the reference computes them (losses.py:37-61,80-85), through the
                tests' fp32 restatement: [B, A, S, S] fp32 scores, where, LogSoftmax, Softmax, KLDivLoss(batchmean) / (A*S),
                torch autograd.  Its score products run as fp32 matmuls (TF32 off, torch's default); the reference's scores come out
                of its attention under autocast, so this leg's products cost more than the reference's would.

Each leg reports ms/step, samples/s and peak allocated memory (over the eager warm-up steps, as a replay's allocations live in the
graph's pool); the card's name and power limit are read in the same run.  --profile adds a
torch.profiler run of the fused step instead of the timings (run it on its own) with the distillation kernels' device time per step.
Writes <out>/bench_distill.json (or bench_distill_profile.json)."""
import argparse
import json
import math
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from deeplearningexamples_b200 import distill as D, ops, training as T  # noqa: E402
from test_distill_cpu import attention_kl, value_kl  # noqa: E402

BACKBONE = {"distillation": True,
            "distillation_config": {"use_attention_scores": True, "use_hidden_states": True, "use_value_states": True,
                                    "use_embedding_states": False, "use_pred_states": False, "attention_loss": "kld",
                                    "hidden_state_loss": "cosine", "embedding_state_loss": "cosine", "value_state_loss": "kld",
                                    "student_teacher_layer_mapping": "last_layer"}}
BASE = dict(hidden_size=768, num_hidden_layers=12, num_attention_heads=12, intermediate_size=3072, vocab_size=30528,
            max_position_embeddings=512, type_vocab_size=2, hidden_act="gelu", initializer_range=0.02,
            hidden_dropout_prob=0.1, attention_probs_dropout_prob=0.1)
STUDENT = dict(BASE, num_hidden_layers=6)              # distillation/BERT_6L_768D/config.json


def gpu_info():
    """Name and power limit of the card the run is on (a read-only nvidia-smi query)."""
    info = dict(gpu=torch.cuda.get_device_name())
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
        info.update(power_limit=q.split(", ")[0], max_sm_clock=q.split(", ")[1])
    except Exception as e:
        info.update(power_limit=f"unknown ({e})")
    return info


class MaterialisedLosses(D.TransformerLosses):
    """The KL losses through the fp32 restatement the tests pin to the reference's own losses.py (tests/test_distill_cpu.py, checked
    against bert_distill_golden.pt): materialised [B, A, S, S] fp32 scores, where, LogSoftmax, Softmax, KLDivLoss(batchmean) / (A*S).
    Cosine as in the fused step."""

    def compute_loss_(self, pred, target, loss_name):
        if loss_name == "attention_loss":
            return attention_kl(pred.materialize(), target.materialize())
        if loss_name == "value_state_loss":
            A = pred.shape[-1] // 64
            return value_kl(pred, target, A, A, pred.shape[1])
        return super().compute_loss_(pred, target, loss_name)


def run_leg(B, S, steps, warmup, materialised):
    dev = torch.device("cuda", 0)
    ops.manual_seed(1)
    student, teacher, project, losses, opt, sch = D.prepare_distill_models_and_optimizer(STUDENT, BASE, dev, BACKBONE,
                                                                                         total_steps=1000)
    if materialised:
        losses = MaterialisedLosses(losses.student_config, losses.teacher_config, dev, None)
    student.train(); teacher.train()
    g = torch.Generator().manual_seed(2)
    batch = {"input_ids": torch.randint(1000, 30522, (B, S), generator=g).to(dev),
             "token_type_ids": (torch.arange(S)[None, :] >= S // 2).long().expand(B, S).contiguous().to(dev),
             "attention_mask": torch.ones(B, S, dtype=torch.long, device=dev)}
    out = {}

    def step():
        out["r"] = D.general_distill_step(student, teacher, project, losses, opt, sch, batch)

    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    graph = T.capture_step_graph(step, warmup_iters=warmup)      # the warm-ups run eagerly: their peak is the step's
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated()
    graph.replay()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        graph.replay()
    torch.cuda.synchronize()
    dt = (time.perf_counter() - t0) / steps
    loss = [x.item() for x in out["r"]]
    res = dict(B=B, S=S, ms_per_step=dt * 1e3, samples_per_s=B / dt, peak_alloc_gib=peak / 2 ** 30,
               loss=loss[0], att_loss=loss[1], rep_loss=loss[2], value_loss=loss[3], finite=all(math.isfinite(x) for x in loss))
    del graph, student, teacher, opt, sch, losses, out
    torch.cuda.empty_cache()
    return res


def profile_fused(B, S, steps):
    dev = torch.device("cuda", 0)
    ops.manual_seed(1)
    student, teacher, project, losses, opt, sch = D.prepare_distill_models_and_optimizer(STUDENT, BASE, dev, BACKBONE, total_steps=1000)
    student.train(); teacher.train()
    batch = {"input_ids": torch.randint(1000, 30522, (B, S), device=dev), "token_type_ids": torch.zeros(B, S, dtype=torch.long, device=dev),
             "attention_mask": torch.ones(B, S, dtype=torch.long, device=dev)}
    for _ in range(3):
        D.general_distill_step(student, teacher, project, losses, opt, sch, batch)
    torch.cuda.synchronize()
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            D.general_distill_step(student, teacher, project, losses, opt, sch, batch)
        torch.cuda.synchronize()
    kern = {}
    total = 0.0
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
        if e.key.startswith("void") or "kernel" in e.key:
            total += t
        if "relkl" in e.key or "sum_partials" in e.key or "cosine_rows" in e.key or "add_rows_bf16" in e.key:
            kern[e.key.split("(")[0].replace("void ", "")] = dict(us_per_step=t / steps, calls_per_step=e.count / steps)
    return dict(B=B, S=S, kernels=kern, all_kernels_us_per_step=total / steps)


ap = argparse.ArgumentParser()
ap.add_argument("--batch", type=int, default=32)
ap.add_argument("--steps", type=int, default=20)
ap.add_argument("--warmup", type=int, default=3)
ap.add_argument("--seqs", default="128,512")
ap.add_argument("--profile", action="store_true", help="only the torch.profiler run of the fused step (run it on its own)")
ap.add_argument("--out", default="bench_out")
args = ap.parse_args()
if not torch.cuda.is_available():
    raise SystemExit("bench_distill needs a GPU")
result = dict(gpu_info(), legs=[])
for S in ([] if args.profile else (int(s) for s in args.seqs.split(","))):
    for materialised in (False, True):
        r = run_leg(args.batch, S, args.steps, args.warmup, materialised)
        r["leg"] = "materialised" if materialised else "fused"
        print(json.dumps(r), flush=True)
        result["legs"].append(r)
if args.profile:
    result["profile"] = [profile_fused(args.batch, int(s), 5) for s in args.seqs.split(",")]
    print(json.dumps(result["profile"]), flush=True)
os.makedirs(args.out, exist_ok=True)
with open(os.path.join(args.out, "bench_distill_profile.json" if args.profile else "bench_distill.json"), "w") as fh:
    json.dump(result, fh, indent=1)
print(json.dumps({k: v for k, v in result.items() if k != "legs"}))
