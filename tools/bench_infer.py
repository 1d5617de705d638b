"""Encoder-only inference throughput (BASELINE.json configs[4]: BERT-large, S=512, B=256, bf16, eval mode, 1xH100):
embeddings + 24 encoder layers + pooler, forward only, CUDA-event timed, eager and as a replayed CUDA graph; full-length batch and a
variable-length batch (lengths ~ U{S/4..S} rounded up to 64, SURVEY.md 8d) where the attention kernel skips fully padded key tiles.
FasterTransformer is a README stub in the reference (SURVEY.md 0), so the parity target for this config is the reference BertModel in
eval mode = the CPU oracle (tests/test_model_gpu.py::test_forward_vs_cpu_oracle_other_shapes, tests/test_attention_gpu.py)."""
import json, os, sys
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from deeplearningexamples_b200 import modeling, training as T

B, S = int(os.environ.get("B", 256)), int(os.environ.get("S", 512))
cfg = dict(T.BERT_LARGE); cfg["vocab_size"] = 30528
torch.manual_seed(0)
model = modeling.BertModel(modeling.BertConfig.from_dict(cfg)).cuda().to(torch.bfloat16).eval()
L_, H, I = 24, 1024, 4096
fwd = L_ * (6 * S * H * H + 4 * S * S * H + 2 * S * H * H + 4 * S * H * I)
out = dict(workload=f"BERT-large encoder-only inference seq{S} bs{B} bf16", runs=[])
for name, full in (("full-length", True), ("variable-length", False)):
    batch = T.synthetic_batch(B, S, cfg["vocab_size"], 1, seed=1, full_mask=full, device="cuda")
    def step():
        with torch.no_grad():
            return model(batch["input_ids"], batch["token_type_ids"], batch["attention_mask"])
    for graphs in (False, True):
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
        ms = e0.elapsed_time(e1) / n
        tokens = int(batch["attention_mask"].sum().item())
        out["runs"].append(dict(batch=name, cuda_graph=graphs, ms_per_batch=round(ms, 2), sequences_per_s=round(B / ms * 1e3, 1),
                                padded_tflops=round(B * fwd / ms / 1e9, 1), real_tokens_per_s=round(tokens / ms * 1e3), token_fill=round(tokens / (B * S), 3)))
        print(out["runs"][-1], flush=True)
print(json.dumps(out))
os.makedirs("bench_out", exist_ok=True); json.dump(out, open("bench_out/bench_infer.json", "w"))
