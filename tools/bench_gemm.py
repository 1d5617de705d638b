"""Microbenchmark of the wgmma GEMM at the BERT-large shapes (fwd / dgrad / wgrad), CUDA-event timed,
inputs larger than L2 are rotated between iterations.  Prints TFLOP/s and fraction of the measured
cuBLAS bf16 peak (MEASURED_PEAKS.json) and times torch.matmul (cuBLAS) beside it on the same shapes."""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from deeplearningexamples_b200 import kernels as k, _lib as L  # noqa: E402


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
    peaks = {}
    p = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "MEASURED_PEAKS.json")
    if os.path.exists(p):
        peaks = json.load(open(p))
    peak = peaks.get("bf16_tflops", 989.0)
    T = int(os.environ.get("T", 16384))
    H, I = 1024, 4096
    rows = []
    bf = torch.bfloat16
    x = torch.randn(T, H, device="cuda").to(bf)
    xi = torch.randn(T, I, device="cuda").to(bf)
    dy3 = torch.randn(T, 3 * H, device="cuda").to(bf)
    w_qkv = (torch.randn(3 * H, H, device="cuda") * 0.02).to(bf)
    w_o = (torch.randn(H, H, device="cuda") * 0.02).to(bf)
    w_1 = (torch.randn(I, H, device="cuda") * 0.02).to(bf)
    w_2 = (torch.randn(H, I, device="cuda") * 0.02).to(bf)
    b_i = torch.zeros(I, device="cuda", dtype=bf)
    cases = [
        ("fwd qkv  [T,H]x[3H,H]", lambda: k.gemm(x, w_qkv), lambda: x @ w_qkv.t(), 2 * T * H * 3 * H),
        ("fwd out  [T,H]x[H,H]", lambda: k.gemm(x, w_o), lambda: x @ w_o.t(), 2 * T * H * H),
        ("fwd ffn1 +bias+gelu", lambda: k.gemm(x, w_1, bias=b_i, epilogue=L.EPI_BIAS_GELU), lambda: x @ w_1.t(), 2 * T * H * I),
        ("fwd ffn2 [T,I]x[H,I]", lambda: k.gemm(xi, w_2), lambda: xi @ w_2.t(), 2 * T * H * I),
        ("dgrad ffn2 dy[T,H]·W2[H,I]", lambda: k.gemm(x, w_2, b_layout=L.LAYOUT_MN), lambda: x @ w_2, 2 * T * H * I),
        ("dgrad ffn1 dy[T,I]·W1[I,H]", lambda: k.gemm(xi, w_1, b_layout=L.LAYOUT_MN), lambda: xi @ w_1, 2 * T * H * I),
        ("dgrad qkv dy[T,3H]·W[3H,H]", lambda: k.gemm(dy3, w_qkv, b_layout=L.LAYOUT_MN), lambda: dy3 @ w_qkv, 2 * T * H * 3 * H),
    ]
    for tn in (0, 128):
        cases.append((f"fwd out tile_n={tn or 256}", lambda tn=tn: k.gemm(x, w_o, tile_n=tn), None, 2 * T * H * H))
        cases.append((f"fwd out +drop+res tile_n={tn or 256}", lambda tn=tn: k.gemm(x, w_o, bias=b_i[:H], aux=x, epilogue=L.EPI_BIAS_DROPOUT_RESIDUAL, dropout_p=0.1, seed=1, tile_n=tn), None, 2 * T * H * H))
        cases.append((f"fwd ffn2 +drop+res tile_n={tn or 256}", lambda tn=tn: k.gemm(xi, w_2, bias=b_i[:H], aux=x, epilogue=L.EPI_BIAS_DROPOUT_RESIDUAL, dropout_p=0.1, seed=1, tile_n=tn), None, 2 * T * H * I))
        cases.append((f"dgrad ffn1 tile_n={tn or 256}", lambda tn=tn: k.gemm(xi, w_1, b_layout=L.LAYOUT_MN, tile_n=tn), None, 2 * T * H * I))
        cases.append((f"dgrad out tile_n={tn or 256}", lambda tn=tn: k.gemm(x, w_o, b_layout=L.LAYOUT_MN, tile_n=tn), None, 2 * T * H * H))
    u = torch.randn(T, I, device="cuda").to(bf)
    cs = torch.zeros(I, device="cuda")
    cases.append(("dgrad ffn2 *gelu'(u) +colsum", lambda: k.gemm(x, w_2, b_layout=L.LAYOUT_MN, aux=u, epilogue=L.EPI_DGELU, colsum_out=cs), None, 2 * T * H * I))
    cases.append(("dgrad ffn1 +add", lambda: k.gemm(xi, w_1, b_layout=L.LAYOUT_MN, aux=x, epilogue=L.EPI_ADD), None, 2 * T * H * I))
    cases.append(("dgrad qkv +add", lambda: k.gemm(dy3, w_qkv, b_layout=L.LAYOUT_MN, aux=x, epilogue=L.EPI_ADD), None, 2 * T * H * 3 * H))
    only = os.environ.get("CASES", "")
    if only == "epi":          # the epilogue-heavy subset (A/B runs of epilogue changes)
        cases = [c for c in cases if any(t in c[0] for t in ("gelu", "drop+res tile_n=256", "+add", "fwd qkv", "fwd out  "))]
    for splits in ((1, 2, 4, 8) if only != "epi" else ()):
        cases.append((f"wgrad ffn1 dy[T,I]^T·x[T,H] splits={splits}",
                      lambda s=splits: k.gemm(xi, x, a_layout=L.LAYOUT_MN, b_layout=L.LAYOUT_MN, epilogue=L.EPI_ATOMIC_F32, splits=s,
                                              out=torch.zeros(I, H, device="cuda")),
                      (lambda: xi.t() @ x) if splits == 1 else None, 2 * T * H * I))
    for splits in ((1, 4, 8, 16) if only != "epi" else ()):
        cases.append((f"wgrad out dy[T,H]^T·x[T,H] splits={splits}",
                      lambda s=splits: k.gemm(x, x, a_layout=L.LAYOUT_MN, b_layout=L.LAYOUT_MN, epilogue=L.EPI_ATOMIC_F32, splits=s,
                                              out=torch.zeros(H, H, device="cuda")),
                      (lambda: x.t() @ x) if splits == 1 else None, 2 * T * H * H))
    exact = os.environ.get("ONLY", "")
    if exact:                  # one case, e.g. under ncu
        cases = [c for c in cases if c[0] == exact]
    for name, ours, ref, flops in cases:
        ms = timeit(ours)
        ms_ref = timeit(ref) if ref is not None else float("nan")
        rows.append(dict(case=name, ms=round(ms, 4), tflops=round(flops / ms / 1e9, 1), frac_of_measured_peak=round(flops / ms / 1e9 / peak, 3),
                         cublas_ms=round(ms_ref, 4), cublas_tflops=round(flops / ms_ref / 1e9, 1) if ref else None))
        print(rows[-1], flush=True)
    os.makedirs("bench_out", exist_ok=True)
    json.dump(dict(T=T, peak_tflops=peak, rows=rows), open("bench_out/bench_gemm.json", "w"), indent=1)


if __name__ == "__main__":
    main()
