"""Encoder-only inference throughput (BASELINE.json configs[4]: BERT-large, S=512, B=256, bf16, eval mode, 1xH100):
embeddings + 24 encoder layers + pooler, forward only, CUDA-event timed.  A full-length batch and a variable-length batch (lengths
~ U{S/4..S} rounded up to 64, SURVEY.md 8d), each on the padded path eager and as a replayed CUDA graph; the padded path runs every
GEMM, LayerNorm and GELU over all B*S rows and attention over all S keys, padding included.  On the variable-length batch the
padding-free route (BertModel.remove_padding: packed tokens, variable-length attention) runs eagerly -- it reads the mask on the
host, so it is not graph-capturable -- alternating with the padded eager leg, three runs each.
FasterTransformer is a README stub in the reference (SURVEY.md 0), so the parity target for this config is the reference BertModel in
eval mode = the CPU oracle (tests/test_model_gpu.py::test_forward_vs_cpu_oracle_other_shapes, tests/test_infer_packed_gpu.py)."""
import json, os, subprocess, sys
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from deeplearningexamples_b200 import modeling, training as T


def gpu_info():
    """Name and power limit of the card the run is on (read-only nvidia-smi query)."""
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


B, S = int(os.environ.get("B", 256)), int(os.environ.get("S", 512))
cfg = dict(T.BERT_LARGE); cfg["vocab_size"] = 30528
torch.manual_seed(0)
model = modeling.BertModel(modeling.BertConfig.from_dict(cfg)).cuda().to(torch.bfloat16).eval()
L_, H, I = 24, 1024, 4096
fwd = L_ * (6 * S * H * H + 4 * S * S * H + 2 * S * H * H + 4 * S * H * I)
out = dict(workload=f"BERT-large encoder-only inference seq{S} bs{B} bf16", **gpu_info(), runs=[])
print(json.dumps({k: v for k, v in out.items() if k != "runs"}), flush=True)


def measure(name, batch, graphs, padding_free, rep=None):
    model.remove_padding(padding_free)

    def step():
        with torch.no_grad():
            return model(batch["input_ids"], batch["token_type_ids"], batch["attention_mask"])
    run = step
    if graphs:
        g = T.capture_step_graph(step, warmup_iters=3)
        run = g.replay
    for _ in range(3): run()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    n = 8
    e0.record()
    for _ in range(n): run()
    e1.record(); torch.cuda.synchronize()
    model.remove_padding(False)
    ms = e0.elapsed_time(e1) / n
    tokens = int(batch["attention_mask"].sum().item())
    r = dict(batch=name, route="padding-free" if padding_free else "padded", cuda_graph=graphs, ms_per_batch=round(ms, 2),
             sequences_per_s=round(B / ms * 1e3, 1), padded_tflops=round(B * fwd / ms / 1e9, 1),
             real_tokens_per_s=round(tokens / ms * 1e3), token_fill=round(tokens / (B * S), 3))
    if rep is not None:
        r["run"] = rep
    out["runs"].append(r)
    print(r, flush=True)


full = T.synthetic_batch(B, S, cfg["vocab_size"], 1, seed=1, full_mask=True, device="cuda")
var = T.synthetic_batch(B, S, cfg["vocab_size"], 1, seed=1, full_mask=False, device="cuda")
for graphs in (False, True):
    measure("full-length", full, graphs, False)
measure("variable-length", var, True, False)
for rep in range(3):                                    # padded and padding-free eager legs alternate
    measure("variable-length", var, False, False, rep)
    measure("variable-length", var, False, True, rep)
print(json.dumps(out))
os.makedirs("bench_out", exist_ok=True); json.dump(out, open("bench_out/bench_infer.json", "w"))
