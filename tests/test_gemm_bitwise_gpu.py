"""GPU: the GEMM's results pinned bit for bit, so that a change to the kernel's code generation that must not change its arithmetic
(register allocation, epilogue data movement, scheduling) is checked exactly rather than within a tolerance.  Every layout pair x
both tile widths x every epilogue, at shapes that hit the edges: one row tile (M < 128) with ragged N (8 valid columns in the last
256-wide tile) and K, an odd number of ragged row tiles, and more tiles than CTAs.  Inputs come from CPU generators, so the outputs
are a function of the kernel alone; their SHA-256 digests are in tests/golden/gemm_bitwise_digests.json
(tests/golden/make_gemm_bitwise_golden.py).  The fp32-atomic epilogue runs with one split, where each output element receives a
single atomic add onto zero; the column sums (atomics across warps, order not fixed) are checked against the pinned output."""
import hashlib
import json
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "gemm_bitwise_digests.json")

LAYOUTS = ["kk", "kmn", "mnmn", "mnk"]      # A layout, B layout: k = K-major, mn = MN-major
TILES = [128, 256]
SHAPES = [(40, 264, 72), (1096, 800, 200), (8320, 1024, 128)]
EPILOGUES = ["bias", "plain_alpha", "gelu", "drop_res", "dgelu_colsum", "add", "tanh", "f32", "atomic"]


def _k():
    from deeplearningexamples_b200 import kernels, _lib
    return kernels, _lib


def _rand(shape, scale, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).to(torch.bfloat16).cuda()


def run_case(layout, bn, shape, epi):
    """The outputs of one case: name -> tensor."""
    k, L = _k()
    M, N, K = shape
    seed = 1000 * LAYOUTS.index(layout) + 100 * SHAPES.index(shape) + 10 * EPILOGUES.index(epi) + bn
    a_mn, b_mn = layout.startswith("mn"), layout.endswith("mn")
    a = _rand((K, M) if a_mn else (M, K), 1.0, seed)
    b = _rand((K, N) if b_mn else (N, K), 0.1, seed + 1)
    kw = dict(a_layout=L.LAYOUT_MN if a_mn else L.LAYOUT_K, b_layout=L.LAYOUT_MN if b_mn else L.LAYOUT_K, tile_n=bn if bn == 128 else 0)
    bias = _rand((N,), 1.0, seed + 2)
    aux = _rand((M, N), 1.5, seed + 3)
    if epi == "bias":
        return {"out": k.gemm(a, b, bias=bias, **kw)}
    if epi == "plain_alpha":
        return {"out": k.gemm(a, b, alpha=0.5, **kw)}
    if epi == "gelu":
        g, u = k.gemm(a, b, bias=bias, epilogue=L.EPI_BIAS_GELU, **kw)
        return {"out": g, "out2": u}
    if epi == "drop_res":
        p = 0.1 if N % 32 == 0 else 0.0                  # dropout works on 32-column groups
        return {"out": k.gemm(a, b, bias=bias, aux=aux, epilogue=L.EPI_BIAS_DROPOUT_RESIDUAL, dropout_p=p, seed=1234 + seed,
                              dropout_stream=3, **kw)}
    if epi == "dgelu_colsum":
        cs = torch.zeros(N, device="cuda")
        out = k.gemm(a, b, aux=aux, epilogue=L.EPI_DGELU, colsum_out=cs, **kw)
        return {"out": out, "colsum": cs}
    if epi == "add":
        return {"out": k.gemm(a, b, aux=aux, epilogue=L.EPI_ADD, **kw)}
    if epi == "tanh":
        return {"out": k.gemm(a, b, bias=bias, epilogue=L.EPI_BIAS_TANH, **kw)}
    if epi == "f32":
        return {"out": k.gemm(a, b, bias=bias, epilogue=L.EPI_F32, **kw)}
    if epi == "atomic":
        return {"out": k.gemm(a, b, epilogue=L.EPI_ATOMIC_F32, splits=1, **kw)}
    raise ValueError(epi)


def case_id(layout, bn, shape, epi):
    return f"{layout}-bn{bn}-{shape[0]}x{shape[1]}x{shape[2]}-{epi}"


def digest(t):
    return hashlib.sha256(t.detach().contiguous().cpu().view(torch.uint8).numpy().tobytes()).hexdigest()


def all_digests():
    res = {}
    for layout in LAYOUTS:
        for bn in TILES:
            for shape in SHAPES:
                for epi in EPILOGUES:
                    outs = run_case(layout, bn, shape, epi)
                    res[case_id(layout, bn, shape, epi)] = {n: digest(t) for n, t in outs.items() if n != "colsum"}
    return res


@pytest.fixture(scope="module")
def golden():
    with open(GOLDEN) as f:
        return json.load(f)


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: f"{s[0]}x{s[1]}x{s[2]}")
@pytest.mark.parametrize("bn", TILES)
@pytest.mark.parametrize("layout", LAYOUTS)
def test_bitwise_against_golden(golden, layout, bn, shape):
    for epi in EPILOGUES:
        cid = case_id(layout, bn, shape, epi)
        outs = run_case(layout, bn, shape, epi)
        for name, want in golden[cid].items():
            assert digest(outs[name]) == want, f"{cid}: {name} differs from the pinned result"
        if "colsum" in outs:
            o = outs["out"].float()
            torch.testing.assert_close(outs["colsum"], o.sum(0), rtol=1e-3, atol=1e-2 * o.abs().sum(0).max().item() + 1e-3)
