"""Where the time of one training step goes: the default bench.py workload (BERT-large phase-2 pretraining, S=512, micro-batch 128,
dropout 0.1, one GPU) run eagerly for a few steps under torch.profiler with CUDA activities.  Writes per-kernel total device time
and share of the step to OUT/step_profile.json and prints the top kernels.

    python tools/step_profile.py [--out bench_out/step_profile] [--steps 3] [--warmup 2] [--batch 128] [--seq 512]
"""
import argparse
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join("bench_out", "step_profile"))
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--batch", type=int, default=128)
    ap.add_argument("--seq", type=int, default=512)
    ap.add_argument("--max-pred", type=int, default=80)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("step_profile.py needs a GPU")
    from torch.profiler import ProfilerActivity, profile

    from deeplearningexamples_b200 import _lib as L
    from deeplearningexamples_b200 import ops
    from deeplearningexamples_b200 import training as T

    device = torch.device("cuda", 0)
    torch.cuda.set_device(device)
    L.load()
    cfg = dict(T.BERT_LARGE)
    cfg["vocab_size"] = 30528
    B, S, P = args.batch, args.seq, args.max_pred
    ops.manual_seed(42)
    model, opt, scaler, sched, crit, _ = T.prepare_model_and_optimizer(cfg, device, distributed=False, seed=42, static_masked_count=B * P)
    model.train()
    batch = {k: v.to(device) for k, v in T.synthetic_batch(B, S, cfg["vocab_size"], P, seed=42).items()}
    loss_acc = torch.zeros(1, dtype=torch.float32, device=device)

    def step():
        T.take_training_step(scaler, model, crit, batch, loss_acc)
        T.take_optimizer_step(sched, opt, scaler)

    for _ in range(args.warmup):
        step()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        t0 = time.perf_counter()
        for _ in range(args.steps):
            step()
        torch.cuda.synchronize()
        wall = time.perf_counter() - t0
    kernels = {}
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            k = kernels.setdefault(e.name, {"calls": 0, "us": 0.0})
            k["calls"] += 1
            k["us"] += e.device_time_total
    busy = sum(k["us"] for k in kernels.values())
    rows = sorted(({"kernel": n, "calls_per_step": k["calls"] / args.steps, "ms_per_step": k["us"] / 1e3 / args.steps,
                    "share_of_device_time": k["us"] / busy} for n, k in kernels.items()), key=lambda r: -r["ms_per_step"])
    attn = [r for r in rows if "dle::attn_" in r["kernel"]]
    props = torch.cuda.get_device_properties(device)
    res = {"gpu": props.name, "workload": f"BERT-large pretraining step, B={B} S={S} max_pred={P}, dropout 0.1, eager, 1 GPU",
           "steps": args.steps, "device_busy_ms_per_step": busy / 1e3 / args.steps, "wall_ms_per_step_profiled": 1e3 * wall / args.steps,
           "attention_ms_per_step": sum(r["ms_per_step"] for r in attn), "attention_share": sum(r["share_of_device_time"] for r in attn),
           "kernels": rows}
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "step_profile.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(f"{props.name}: device busy {res['device_busy_ms_per_step']:.1f} ms/step, attention {res['attention_ms_per_step']:.1f} ms "
          f"({100 * res['attention_share']:.1f} %)")
    for r in rows[:25]:
        print(f"  {r['ms_per_step']:8.2f} ms  {100 * r['share_of_device_time']:5.1f} %  x{r['calls_per_step']:.0f}  {r['kernel'][:110]}")


if __name__ == "__main__":
    main()
