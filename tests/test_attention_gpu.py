"""GPU parity: fused attention fwd/bwd vs a plain torch fp32 restatement of
BertSelfAttention (modeling.py:349-376) on the same bf16 inputs."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu
bf = torch.bfloat16


def _k():
    from deeplearningexamples_b200 import kernels
    return kernels


def ref_attention(qkv, mask, B, S, A, drop_mask=None, p=0.0):
    """fp32 reference.  qkv [B*S,3H] (any float dtype, autograd ok); mask [B,S] additive or None;
    drop_mask [B,A,S,S] bool keep-mask or None.  Returns ctx [B*S,H], lse [B,A,S]."""
    H = A * 64
    x = qkv.float().view(B, S, 3, A, 64)
    q, k, v = (x[:, :, i].permute(0, 2, 1, 3) for i in range(3))          # [B,A,S,64]
    s = q @ k.transpose(-1, -2) / math.sqrt(64)
    if mask is not None:
        s = s + mask.float().view(B, 1, 1, S)
    lse = torch.logsumexp(s, dim=-1)
    pr = torch.softmax(s, dim=-1)
    if drop_mask is not None:
        pr = pr * drop_mask / (1 - p)
    ctx = (pr @ v).permute(0, 2, 1, 3).reshape(B * S, H)
    return ctx, lse


def _inputs(B, S, A, seed, ragged):
    g = torch.Generator(device="cuda").manual_seed(seed)
    qkv = (torch.randn(B * S, 3 * A * 64, generator=g, device="cuda") * 1.0).to(bf)
    mask = None
    if ragged:
        lens = torch.randint(S // 4, S + 1, (B,), generator=g, device="cuda")
        lens[0] = S
        keep = (torch.arange(S, device="cuda").unsqueeze(0) < lens.unsqueeze(1)).float()
        mask = (1.0 - keep) * -10000.0
    return qkv, mask


@pytest.mark.parametrize("B,S,A", [(1, 128, 1), (2, 128, 4), (2, 256, 2), (1, 384, 3), (3, 512, 2), (2, 512, 16)])
@pytest.mark.parametrize("ragged", [False, True])
def test_attention_forward(B, S, A, ragged):
    k = _k()
    qkv, mask = _inputs(B, S, A, seed=B * 1000 + S + A, ragged=ragged)
    ctx, lse = k.attn_fwd(qkv, mask, B, S, A)
    ctx_ref, lse_ref = ref_attention(qkv, mask, B, S, A)
    torch.testing.assert_close(lse, lse_ref, rtol=1e-3, atol=2e-3)
    torch.testing.assert_close(ctx.float(), ctx_ref, rtol=2e-2, atol=2e-2)


@pytest.mark.parametrize("B,S,A", [(1, 128, 1), (2, 128, 4), (2, 256, 2), (1, 384, 3), (2, 512, 2), (1, 512, 16)])
@pytest.mark.parametrize("ragged", [False, True])
def test_attention_backward(B, S, A, ragged):
    k = _k()
    qkv, mask = _inputs(B, S, A, seed=7 * B + S + A, ragged=ragged)
    g = torch.Generator(device="cuda").manual_seed(99)
    dctx = torch.randn(B * S, A * 64, generator=g, device="cuda").to(bf)
    ctx, lse = k.attn_fwd(qkv, mask, B, S, A)
    dbias = torch.zeros(3 * A * 64, device="cuda")
    dqkv = k.attn_bwd(qkv, mask, ctx, dctx, lse, B, S, A, dbias=dbias)
    # fused q/k/v bias gradients == column sums of the dqkv the kernel stored
    torch.testing.assert_close(dbias, dqkv.float().sum(0), rtol=1e-3, atol=2e-2 * max(1.0, dqkv.float().abs().max().item()))
    x = qkv.float().requires_grad_(True)
    ctx_ref, _ = ref_attention(x, mask, B, S, A)
    ctx_ref.backward(dctx.float())
    ref = x.grad
    # bf16 P/dS operands: compare with a tolerance relative to the gradient scale of each q/k/v block
    H = A * 64
    for i, name in enumerate("qkv"):
        got, want = dqkv[:, i * H:(i + 1) * H].float(), ref[:, i * H:(i + 1) * H]
        err = (got - want).abs().max().item()
        assert err <= 2e-2 * want.abs().max().item() + 1e-3, (name, err, want.abs().max().item())
        cos = torch.nn.functional.cosine_similarity(got.flatten(), want.flatten(), dim=0).item()
        assert cos > 0.999, (name, cos)


def _extract_keep_mask(k, qkv, mask, B, S, A, p, seed, stream):
    """Recover the exact dropout keep-mask of the fused kernel: P~[q, key] = ctx[q, d] when V is a slab of the
    identity (V[key, d] = 1 iff key == c*64 + d)."""
    H = A * 64
    probs = torch.zeros(B, A, S, S, device="cuda")
    for c in range(S // 64):
        q2 = qkv.clone()
        v = torch.zeros(B, S, A, 64, device="cuda")
        idx = torch.arange(64, device="cuda")
        v[:, c * 64 + idx, :, idx] = 1.0
        q2[:, 2 * H:] = v.view(B * S, H).to(bf)
        ctx, _ = k.attn_fwd(q2, mask, B, S, A, dropout_p=p, seed=seed, dropout_stream=stream)
        probs[:, :, :, c * 64:(c + 1) * 64] = ctx.float().view(B, S, A, 64).permute(0, 2, 1, 3)
    return probs


def test_attention_dropout_fwd_bwd_consistent():
    k = _k()
    B, S, A, p, seed, stream = 2, 256, 2, 0.1, 4242, 3
    qkv, mask = _inputs(B, S, A, seed=5, ragged=True)
    qkv = (qkv.float() * 0.5).to(bf)                    # keep probabilities well away from bf16 underflow
    pd = _extract_keep_mask(k, qkv, mask, B, S, A, p, seed, stream)
    _, lse = k.attn_fwd(qkv, mask, B, S, A)
    # P (no dropout) from reference; keep-mask = where the dropped P~ is non-zero
    x = qkv.float().view(B, S, 3, A, 64)
    q, kk = x[:, :, 0].permute(0, 2, 1, 3), x[:, :, 1].permute(0, 2, 1, 3)
    s = q @ kk.transpose(-1, -2) / 8 + (mask.view(B, 1, 1, S) if mask is not None else 0)
    pr = torch.softmax(s, -1)
    valid = pr > 1e-4                                     # positions where P~ cannot underflow to 0 in bf16
    keep = pd > 0
    frac = keep[valid].float().mean().item()
    assert 0.885 < frac < 0.915, frac
    torch.testing.assert_close(pd[valid & keep], (pr / (1 - p))[valid & keep], rtol=3e-2, atol=1e-3)
    # full fwd/bwd with dropout vs autograd using the extracted mask
    keep_full = keep | ~valid                              # where P ~ 0 the mask value is irrelevant
    ctx, lse = k.attn_fwd(qkv, mask, B, S, A, dropout_p=p, seed=seed, dropout_stream=stream)
    xr = qkv.float().requires_grad_(True)
    ctx_ref, _ = ref_attention(xr, mask, B, S, A, drop_mask=keep_full.float(), p=p)
    torch.testing.assert_close(ctx.float(), ctx_ref, rtol=3e-2, atol=3e-2)
    g = torch.Generator(device="cuda").manual_seed(1)
    dctx = torch.randn(B * S, A * 64, generator=g, device="cuda").to(bf)
    dqkv = k.attn_bwd(qkv, mask, ctx, dctx, lse, B, S, A, dropout_p=p, seed=seed, dropout_stream=stream)
    ctx_ref.backward(dctx.float())
    H = A * 64
    for i, name in enumerate("qkv"):
        got, want = dqkv[:, i * H:(i + 1) * H].float(), xr.grad[:, i * H:(i + 1) * H]
        cos = torch.nn.functional.cosine_similarity(got.flatten(), want.flatten(), dim=0).item()
        assert cos > 0.998, (name, cos)
        assert (got - want).abs().max().item() <= 3e-2 * want.abs().max().item() + 1e-3, name
    # different stream => different mask; same stream => bitwise identical
    ctx2, _ = k.attn_fwd(qkv, mask, B, S, A, dropout_p=p, seed=seed, dropout_stream=stream)
    ctx3, _ = k.attn_fwd(qkv, mask, B, S, A, dropout_p=p, seed=seed, dropout_stream=stream + 1)
    assert torch.equal(ctx, ctx2) and not torch.equal(ctx, ctx3)


def test_attention_linear_in_v_full_size():
    """BASELINE-size property (B=8,S=512,A=16 with dropout): ctx is linear in V, so <dctx, ctx> == <dV, V>."""
    k = _k()
    B, S, A, p = 8, 512, 16, 0.1
    qkv, mask = _inputs(B, S, A, seed=11, ragged=False)
    H = A * 64
    g = torch.Generator(device="cuda").manual_seed(2)
    dctx = torch.randn(B * S, H, generator=g, device="cuda").to(bf)
    ctx, lse = k.attn_fwd(qkv, mask, B, S, A, dropout_p=p, seed=77, dropout_stream=1)
    dqkv = k.attn_bwd(qkv, mask, ctx, dctx, lse, B, S, A, dropout_p=p, seed=77, dropout_stream=1)
    lhs = (dctx.double() * ctx.double()).sum().item()
    rhs = (dqkv[:, 2 * H:].double() * qkv[:, 2 * H:].double()).sum().item()
    assert abs(lhs - rhs) <= 2e-2 * max(abs(lhs), abs(rhs), 1.0) + 5.0, (lhs, rhs)


def test_attention_skips_fully_padded_key_tiles():
    """Variable-length batches (SURVEY.md 8f rank 3): key tiles whose additive mask is -10000 for every key are skipped outright by
    the kernels; the results must equal the dense computation (fp32 reference) and dK / dV of padded keys must be exactly zero."""
    k = _k()
    B, S, A = 4, 512, 2
    H = A * 64
    g = torch.Generator(device="cuda").manual_seed(21)
    qkv = torch.randn(B * S, 3 * H, generator=g, device="cuda").to(bf)
    lens = torch.tensor([S, 100, 129, 256], device="cuda")
    keep = (torch.arange(S, device="cuda").unsqueeze(0) < lens.unsqueeze(1)).float()
    mask = (1.0 - keep) * -10000.0
    dctx = torch.randn(B * S, H, generator=g, device="cuda").to(bf)
    ctx, lse = k.attn_fwd(qkv, mask, B, S, A)
    ctx_ref, lse_ref = ref_attention(qkv, mask, B, S, A)
    torch.testing.assert_close(lse, lse_ref, rtol=1e-3, atol=2e-3)
    torch.testing.assert_close(ctx.float(), ctx_ref, rtol=2e-2, atol=2e-2)
    dqkv = k.attn_bwd(qkv, mask, ctx, dctx, lse, B, S, A)
    x = qkv.float().requires_grad_(True)
    ref_attention(x, mask, B, S, A)[0].backward(dctx.float())
    for i, name in enumerate("qkv"):
        got, want = dqkv[:, i * H:(i + 1) * H].float(), x.grad[:, i * H:(i + 1) * H]
        assert (got - want).abs().max().item() <= 2e-2 * want.abs().max().item() + 1e-3, name
    pad = (keep.view(-1) == 0)
    assert torch.count_nonzero(dqkv[pad][:, H:]) == 0                      # dK, dV rows of padded keys: exactly zero
    # same bits with the mask given per key but no tile fully padded (exactness of the skip: compare a padded batch row with itself
    # embedded in a batch whose other rows force every tile to be visited)
    ctx2, lse2 = k.attn_fwd(qkv[S:2 * S].contiguous(), mask[1:2].contiguous(), 1, S, A)
    assert torch.equal(ctx2, ctx[S:2 * S]) and torch.equal(lse2, lse[1:2])


def test_attention_rejects_bad_shapes():
    from deeplearningexamples_b200 import _lib
    k = _k()
    qkv = torch.zeros(100, 192, device="cuda", dtype=bf)
    with pytest.raises(_lib.DleError):
        k.attn_fwd(qkv, None, 1, 100, 1)
