"""LAMB microbenchmark on the BERT-large tensor list (398 tensors, 336M params): our 3-launch multi-tensor LAMB vs the
reference's fused_lamb_CUDA kernels (oracle/_ref, driven as fused_lamb.py does), CUDA-event timed.
Algorithmic bytes: 28 B/param (SURVEY.md 8d) -> achieved GB/s and fraction of the measured HBM peak."""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from deeplearningexamples_b200.lamb import FusedLAMBAMP  # noqa: E402
from oracle import bert_oracle as O  # noqa: E402
from oracle import build_ref  # noqa: E402


def timeit(fn, iters=10, warm=3):
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
    peak = 6574.1
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        peak = json.load(open(p))["hbm_gbs"]
    shapes = O.param_shapes(O.BERT_LARGE)
    no_decay = ['bias', 'gamma', 'beta', 'LayerNorm']
    out = {}
    for gdt in (torch.bfloat16, torch.float32):
        decay, nodecay = [], []
        for name, shp in shapes.items():
            q = torch.nn.Parameter((torch.randn(shp, device="cuda") * 0.02).to(gdt))
            q.grad = (torch.randn(shp, device="cuda") * 1e-3).to(gdt)
            (nodecay if any(nd in name for nd in no_decay) else decay).append(q)
        n = sum(q.numel() for q in decay + nodecay)
        opt = FusedLAMBAMP([{'params': decay, 'weight_decay': 0.01}, {'params': nodecay, 'weight_decay': 0.0}], lr=1e-3)
        opt.setup_fp32_params()
        ms = timeit(lambda: opt.step())
        key = "ours_bf16grad_fp32master" if gdt == torch.bfloat16 else "ours_fp32"
        out[key] = dict(ms=round(ms, 4), n_params=n, algorithmic_GBps=round(28 * n / ms / 1e6, 1), frac_of_measured_hbm=round(28 * n / ms / 1e6 / peak, 3), launches=3)
        print(key, out[key], flush=True)
        if gdt == torch.float32:
            ext = build_ref.load_module()
            if ext is not None:
                groups = [(decay, 0.01), (nodecay, 0.0)]
                st = [[(torch.zeros_like(q), torch.zeros_like(q)) for q in g] for g, _ in groups]
                noop = torch.zeros(1, dtype=torch.int, device="cuda")
                steps = [torch.zeros(1, dtype=torch.int, device="cuda") for _ in groups]
                lr = torch.tensor(1e-3, device="cuda")
                found_inf, inv_scale, mx = torch.zeros(1, device="cuda"), torch.ones(1, device="cuda"), torch.ones(1, device="cuda")

                def ref_step():
                    # fused_lamb.py:148-258: inf check sweep, grad norm, blend, then per group l2norm/stage1/l2norm/stage2
                    allg = [q.grad for g, _ in groups for q in g]
                    torch._amp_foreach_non_finite_check_and_unscale_(allg, found_inf, inv_scale)
                    g32 = ext.multi_tensor_l2norm(65536, noop, [allg], False)[0]
                    gn = ext.multi_tensor_l2norm(65536, noop, [[g32, torch.zeros_like(g32)]], False)[0]
                    for (g, wd), s, stp in zip(groups, st, steps):
                        stp += (noop != 1).int()
                        ext.multi_tensor_lamb(65536, noop, [[q.grad for q in g], [q.data for q in g], [a for a, _ in s], [b for _, b in s]],
                                              lr, 0.9, 0.999, 1e-6, stp, 1, wd, 1, 1, gn, mx, False, found_inf, inv_scale)
                ms_r = timeit(ref_step)
                out["reference_fused_lamb_CUDA_fp32"] = dict(ms=round(ms_r, 4), algorithmic_GBps=round(28 * n / ms_r / 1e6, 1),
                                                             frac_of_measured_hbm=round(28 * n / ms_r / 1e6 / peak, 3))
                print("reference", out["reference_fused_lamb_CUDA_fp32"], flush=True)
        del opt, decay, nodecay
        torch.cuda.empty_cache()
    os.makedirs("bench_out", exist_ok=True)
    json.dump(dict(hbm_peak_GBps=peak, **out), open("bench_out/bench_lamb.json", "w"), indent=1)


if __name__ == "__main__":
    main()
