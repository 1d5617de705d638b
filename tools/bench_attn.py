"""Attention microbenchmark (B=32, S=512, A=16 by default): fwd / bwd, with and without dropout / mask, CUDA-event timed."""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from deeplearningexamples_b200 import kernels as k  # noqa: E402


def timeit(fn, iters=20, warm=5):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    B, S, A = int(os.environ.get("B", 32)), int(os.environ.get("S", 512)), int(os.environ.get("A", 16))
    H = A * 64
    qkv = torch.randn(B * S, 3 * H, device="cuda").to(torch.bfloat16)
    dctx = torch.randn(B * S, H, device="cuda").to(torch.bfloat16)
    mask = torch.zeros(B, S, device="cuda")
    rows = []
    for name, m, p in (("nomask,p=0", None, 0.0), ("mask,p=0", mask, 0.0), ("mask,p=0.1", mask, 0.1)):
        ctx, lse = k.attn_fwd(qkv, m, B, S, A, dropout_p=p, seed=1, dropout_stream=1)
        f = timeit(lambda: k.attn_fwd(qkv, m, B, S, A, dropout_p=p, seed=1, dropout_stream=1))
        b = timeit(lambda: k.attn_bwd(qkv, m, ctx, dctx, lse, B, S, A, dropout_p=p, seed=1, dropout_stream=1))
        ff, bf = 4.0 * S * S * 64 * B * A, 10.0 * S * S * 64 * B * A
        rows.append(dict(case=name, fwd_us=round(f * 1e3, 1), fwd_tflops=round(ff / f / 1e9, 1), bwd_us=round(b * 1e3, 1), bwd_tflops=round(bf / b / 1e9, 1)))
        print(rows[-1], flush=True)
    os.makedirs("bench_out", exist_ok=True)
    json.dump(dict(B=B, S=S, A=A, rows=rows), open("bench_out/bench_attn.json", "w"), indent=1)


if __name__ == "__main__":
    main()
