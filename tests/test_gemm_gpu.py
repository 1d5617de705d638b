"""GPU parity: wgmma GEMM (all operand layouts and epilogues) vs a plain torch fp32 reference of the
same op on the same bf16 inputs.  Tolerance: bf16 output rounding (rel 2^-8) + fp32 accumulation order."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _k():
    from deeplearningexamples_b200 import kernels, _lib
    return kernels, _lib


def _rand(shape, scale=1.0, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(shape, generator=g, device="cuda") * scale).to(torch.bfloat16)


def _close(got, want, rtol=1e-2, atol=None):
    want = want.float(); got = got.float()
    atol = atol if atol is not None else 1e-2 * want.abs().max().item() + 1e-6
    torch.testing.assert_close(got, want, rtol=rtol, atol=atol)


SHAPES = [(128, 256, 64), (256, 512, 128), (384, 1024, 1024), (1000, 768, 320), (2048, 4096, 1024), (130, 264, 72)]


@pytest.mark.parametrize("M,N,K", SHAPES)
def test_forward_kk(M, N, K):
    k, L = _k()
    a, b = _rand((M, K), seed=1), _rand((N, K), 0.05, seed=2)
    bias = _rand((N,), seed=3)
    out = k.gemm(a, b, bias=bias)
    _close(out, a.float() @ b.float().t() + bias.float())


@pytest.mark.parametrize("M,N,K", SHAPES)
def test_dgrad_k_mn(M, N, K):
    """dx[M,N] = dy[M,K] @ W[K,N]  (B operand MN-major, read where it lies)."""
    k, L = _k()
    a, w = _rand((M, K), seed=4), _rand((K, N), 0.05, seed=5)
    out = k.gemm(a, w, b_layout=L.LAYOUT_MN)
    _close(out, a.float() @ w.float())


@pytest.mark.parametrize("M,N,K", [(256, 512, 128), (1024, 1024, 2048), (4096, 1024, 4096), (320, 768, 1000), (264, 136, 200)])
@pytest.mark.parametrize("splits", [1, 3, 8])
def test_wgrad_mn_mn_splitk(M, N, K, splits):
    """dW[M,N] = dy[K,M]^T @ x[K,N]  (both operands MN-major), split-K with fp32 red.global.add."""
    k, L = _k()
    dy, x = _rand((K, M), seed=6), _rand((K, N), seed=7)
    out = k.gemm(dy, x, a_layout=L.LAYOUT_MN, b_layout=L.LAYOUT_MN, epilogue=L.EPI_ATOMIC_F32, splits=splits)
    want = dy.float().t() @ x.float()
    torch.testing.assert_close(out, want, rtol=1e-3, atol=1e-3 * want.abs().max().item())


def test_tile128_path():
    k, L = _k()
    a, b = _rand((300, 512), seed=8), _rand((128, 512), 0.05, seed=9)
    _close(k.gemm(a, b), a.float() @ b.float().t())
    b2 = _rand((1024, 512), 0.05, seed=10)
    _close(k.gemm(a, b2, tile_n=128), a.float() @ b2.float().t())


def test_strided_views():
    """operands that are column slices of a wider matrix (ld > cols), as the packed-QKV layout needs."""
    k, L = _k()
    big = _rand((512, 3 * 256), seed=11)
    w = _rand((256, 256), 0.05, seed=12)
    a = big[:, 256:512]
    out_big = torch.zeros((512, 3 * 256), device="cuda", dtype=torch.bfloat16)
    k.gemm(a, w, out=out_big[:, 512:768])
    _close(out_big[:, 512:768], a.float() @ w.float().t())
    assert out_big[:, :512].abs().max().item() == 0.0


def test_epilogue_bias_gelu():
    k, L = _k()
    a, b, bias = _rand((512, 256), seed=13), _rand((1024, 256), 0.1, seed=14), _rand((1024,), seed=15)
    g, u = k.gemm(a, b, bias=bias, epilogue=L.EPI_BIAS_GELU)
    u_ref = a.float() @ b.float().t() + bias.float()
    _close(u, u_ref)
    _close(g, torch.nn.functional.gelu(u.float(), approximate="tanh"), rtol=1e-2, atol=1e-2)


def test_epilogue_dgelu_and_add():
    k, L = _k()
    a, b = _rand((512, 1024), seed=16), _rand((1024, 256), 0.05, seed=17)
    u = _rand((512, 256), 1.5, seed=18)
    out = k.gemm(a, b, b_layout=L.LAYOUT_MN, epilogue=L.EPI_DGELU, aux=u)
    uf = u.float().requires_grad_(True)
    torch.nn.functional.gelu(uf, approximate="tanh").sum().backward()
    _close(out, (a.float() @ b.float()) * uf.grad)
    out2 = k.gemm(a, b, b_layout=L.LAYOUT_MN, epilogue=L.EPI_ADD, aux=u)
    _close(out2, a.float() @ b.float() + u.float())


@pytest.mark.parametrize("M,N,K", [(130, 264, 72), (1000, 776, 320), (4096, 4096, 1024)])
def test_epilogue_dgelu_ragged_and_wide(M, N, K):
    """The gelu'(u) epilogue on the 256-wide tile: partial row tiles, a last column tile with 8 valid columns, and the full FFN width,
    with the column sums."""
    k, L = _k()
    a, w, u = _rand((M, K), seed=50), _rand((K, N), 0.05, seed=51), _rand((M, N), 1.5, seed=52)
    cs = torch.zeros(N, device="cuda")
    out = k.gemm(a, w, b_layout=L.LAYOUT_MN, epilogue=L.EPI_DGELU, aux=u, colsum_out=cs)
    uf = u.float().requires_grad_(True)
    torch.nn.functional.gelu(uf, approximate="tanh").sum().backward()
    _close(out, (a.float() @ w.float()) * uf.grad)
    torch.testing.assert_close(cs, out.float().sum(dim=0), rtol=1e-3, atol=1e-2 * out.float().abs().sum(dim=0).max().item() + 1e-3)


def test_epilogue_dropout_residual_statistics_and_determinism():
    k, L = _k()
    a, b, bias, res = _rand((1024, 256), seed=19), _rand((512, 256), 0.1, seed=20), _rand((512,), seed=21), _rand((1024, 512), seed=22)
    base = a.float() @ b.float().t() + bias.float()
    o0 = k.gemm(a, b, bias=bias, aux=res, epilogue=L.EPI_BIAS_DROPOUT_RESIDUAL, dropout_p=0.0)
    _close(o0, base + res.float())
    o1 = k.gemm(a, b, bias=bias, aux=res, epilogue=L.EPI_BIAS_DROPOUT_RESIDUAL, dropout_p=0.1, seed=1234, dropout_stream=7)
    o2 = k.gemm(a, b, bias=bias, aux=res, epilogue=L.EPI_BIAS_DROPOUT_RESIDUAL, dropout_p=0.1, seed=1234, dropout_stream=7)
    assert torch.equal(o1, o2)
    d = (o1.float() - res.float())
    dropped = (d.abs() < 1e-2 * base.abs().clamp_min(0.5)) & (base.abs() > 0.5)
    frac = dropped.float().sum() / (base.abs() > 0.5).float().sum()
    assert 0.08 < frac.item() < 0.12
    kept = ~dropped & (base.abs() > 0.5)
    torch.testing.assert_close(d[kept], (base / 0.9)[kept], rtol=3e-2, atol=3e-2)


def test_f32_and_tanh_epilogues():
    k, L = _k()
    a, b, bias = _rand((200, 256), seed=23), _rand((512, 256), 0.1, seed=24), _rand((512,), seed=25)
    ref = a.float() @ b.float().t() + bias.float()
    torch.testing.assert_close(k.gemm(a, b, bias=bias, epilogue=L.EPI_F32), ref, rtol=1e-4, atol=1e-3)
    _close(k.gemm(a, b, bias=bias, epilogue=L.EPI_BIAS_TANH), torch.tanh(ref))


def test_linearity_full_size():
    """size-independent property at the BERT-large FFN shape: f(a1+a2) == f(a1)+f(a2) in fp32 output."""
    k, L = _k()
    T, H, I = 4096, 1024, 4096
    a1, a2, w = _rand((T, H), seed=26), _rand((T, H), seed=27), _rand((I, H), 0.02, seed=28)
    s = (a1.float() + a2.float()).to(torch.bfloat16)
    exact = (s.float() == a1.float() + a2.float())          # rows where the bf16 sum is exact
    o1, o2, o3 = (k.gemm(x, w, epilogue=L.EPI_F32) for x in (a1, a2, s))
    rows = exact.all(dim=1)
    assert rows.sum() >= 0
    err = (o3 - (o1 + o2)).abs()
    bound = 0.05 * (~exact).float().sum(dim=1, keepdim=True) * 0.02 * 8 + 1e-3
    assert (err <= bound + 1e-3 * o3.abs()).all()


def test_small_and_ragged_reduction_dims():
    """wgrad of the pooler / MLM head: the reduction dim is a row count (B or N_mask), any value."""
    k, L = _k()
    for rows in (2, 20, 33):
        dy, x = _rand((rows, 256), seed=31), _rand((rows, 512), seed=32)
        out = k.gemm(dy, x, a_layout=L.LAYOUT_MN, b_layout=L.LAYOUT_MN, epilogue=L.EPI_F32)
        torch.testing.assert_close(out, dy.float().t() @ x.float(), rtol=1e-3, atol=1e-2)
    a, w = _rand((20, 264), seed=33), _rand((512, 264), 0.05, seed=34)     # K = 264: partial last k-block
    _close(k.gemm(a, w), a.float() @ w.float().t())
    xs = _rand((4, 128, 256), seed=35)[:, 0]                                # strided rows (hidden_states[:, 0])
    _close(k.gemm(xs, _rand((256, 256), 0.05, seed=36)), xs.float() @ _rand((256, 256), 0.05, seed=36).float().t())


def test_invalid_args_return_error():
    k, L = _k()
    a, b = _rand((128, 60), seed=29), _rand((128, 60), seed=30)   # row stride not a multiple of 16 bytes
    with pytest.raises(L.DleError):
        k.gemm(a, b)
    with pytest.raises(L.DleError):
        k.gemm(a.cpu(), b.cpu())


def test_epilogue_column_sums_of_output():
    """colsum_out: the GEMM accumulates column sums of its (bf16) output -- the bias gradient of the producing layer -- so no
    separate pass re-reads the tensor (warp transpose-reduce + red.global.add)."""
    k, L = _k()
    a, w, u = _rand((1000, 512), seed=40), _rand((512, 768), 0.05, seed=41), _rand((1000, 768), 1.5, seed=42)
    acc = torch.zeros(768, device="cuda")
    out = k.gemm(a, w, b_layout=L.LAYOUT_MN, epilogue=L.EPI_DGELU, aux=u, colsum_out=acc)
    torch.testing.assert_close(acc, out.float().sum(0), rtol=1e-4, atol=2e-2)
    acc2 = torch.zeros(768, device="cuda")
    out2 = k.gemm(a, w, b_layout=L.LAYOUT_MN, colsum_out=acc2)
    torch.testing.assert_close(acc2, out2.float().sum(0), rtol=1e-4, atol=2e-2)


@pytest.mark.parametrize("N,tile_n", [(1024, 0), (512, 128)])
def test_epilogues_many_tiles_per_cta(N, tile_n):
    """Persistent-kernel state that only shows with several tiles per CTA (the encoder shapes run 14+): the bias slice is staged one
    tile ahead and rotates over three shared-memory slots, and the residual / pre-activation operand of a tile's first chunk is
    prefetched by cp.async from the previous tile's last chunk.  16384 x N output = 512 tiles on 132 CTAs, non-zero bias that differs
    per column tile, every epilogue that takes a bias or an aux operand, against fp32 torch."""
    k, L = _k()
    M, K = 16384, 256
    a, w = _rand((M, K), seed=40), _rand((N, K), 0.1, seed=41)
    bias = (_rand((N,), 1.0, seed=42).float() + torch.arange(N, device="cuda").float() / N).to(torch.bfloat16)
    res = _rand((M, N), 1.0, seed=43)
    base = a.float() @ w.float().t()
    _close(k.gemm(a, w, bias=bias, tile_n=tile_n), base + bias.float())
    _close(k.gemm(a, w, bias=bias, aux=res, epilogue=L.EPI_BIAS_DROPOUT_RESIDUAL, dropout_p=0.0, tile_n=tile_n), base + bias.float() + res.float())
    g, u = k.gemm(a, w, bias=bias, epilogue=L.EPI_BIAS_GELU, tile_n=tile_n)
    _close(u, base + bias.float())
    _close(g, torch.nn.functional.gelu(u.float(), approximate="tanh"), rtol=1e-2, atol=1e-2)
    _close(k.gemm(a, w, aux=res, epilogue=L.EPI_ADD, tile_n=tile_n), base + res.float())
    cs = torch.zeros(N, device="cuda")
    out = k.gemm(a, w, aux=res, epilogue=L.EPI_DGELU, colsum_out=cs, tile_n=tile_n)
    rf = res.float().requires_grad_(True)
    torch.nn.functional.gelu(rf, approximate="tanh").sum().backward()
    _close(out, base * rf.grad)
    torch.testing.assert_close(cs, out.float().sum(dim=0), rtol=1e-3, atol=1e-2 * out.float().abs().sum(dim=0).max().item())
