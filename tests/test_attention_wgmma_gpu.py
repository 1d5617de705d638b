"""Fused attention: exact dropout keep-mask and bitwise-reproducible backward.

The keep decision of every (b, h, query, key) is pinned bit for bit to a NumPy restatement of common.cuh (attn_dropout_block,
attn_dropout_word, attn_dropout_k2): the statistical dropout tests would still pass if a change of the MMA fragment layout permuted
mask bits, this one does not."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
bf = torch.bfloat16
M32 = 0xFFFFFFFF


def _philox4x32_7(c0, c1, c2, c3, k0, k1):
    """Philox4x32 with 7 rounds on uint64 arrays holding 32-bit values (common.cuh: philox4x32)."""
    M0, M1, W0, W1 = 0xD2511F53, 0xCD9E8D57, 0x9E3779B9, 0xBB67AE85
    for _ in range(7):
        p0, p1 = np.uint64(M0) * c0, np.uint64(M1) * c2
        hi0, lo0, hi1, lo1 = p0 >> np.uint64(32), p0 & np.uint64(M32), p1 >> np.uint64(32), p1 & np.uint64(M32)
        c0, c1, c2, c3 = hi1 ^ c1 ^ np.uint64(k0), lo1, hi0 ^ c3 ^ np.uint64(k1), lo0
        k0, k1 = (k0 + W0) & M32, (k1 + W1) & M32
    return c0, c1, c2, c3


def _thresh15(p):
    t = np.float32(p) * np.float32(32768.0) + np.float32(0.5)
    return 0 if t <= 0 else (32767 if t >= 32767 else int(t))


def reference_keep(B, S, A, p, seed, stream):
    """bool [B, A, S, S]: element (b, h, q, key) belongs to group32 = ((b*A + h)*S + q)*S + key >> 5; its Philox block gives 16 pair
    words; element 2i | 2i+1 of the group is kept iff bit 15 | bit 31 of word i is set."""
    k2 = ((0x8000 - _thresh15(p)) * 0x00010001) & M32
    groups = np.arange(B * A * S * S // 32, dtype=np.uint64)
    r = _philox4x32_7(groups & np.uint64(M32), groups >> np.uint64(32), np.full_like(groups, stream), np.full_like(groups, 0xA77D20),
                      seed & M32, (seed >> 32) & M32)
    consts = (0x9E3779B1, 0x85EBCA77, 0xC2B2AE3D, 0x27D4EB2F)
    keep = np.empty((groups.size, 32), dtype=bool)
    for i in range(16):
        m = (r[i >> 2] * np.uint64(consts[i & 3])) & np.uint64(M32)
        y = (((m ^ (m >> np.uint64(16))) & np.uint64(0x7FFF7FFF)) + np.uint64(k2)) & np.uint64(M32)
        keep[:, 2 * i] = (y >> np.uint64(15)) & np.uint64(1) == 1
        keep[:, 2 * i + 1] = (y >> np.uint64(31)) & np.uint64(1) == 1
    return keep.reshape(B, A, S, S)


def test_dropout_keep_mask_matches_restatement_bitwise():
    from deeplearningexamples_b200 import kernels as k
    B, S, A, p, seed, stream = 1, 512, 2, 0.1, 0x1234_5678_9ABC, 5
    H = A * 64
    g = torch.Generator(device="cuda").manual_seed(3)
    qkv = (torch.randn(B * S, 3 * H, generator=g, device="cuda") * 0.5).to(bf)
    # P~[q, key] = ctx[q, d] * (1 - p) * l when V is a slab of the identity (V[key, d] = 1 iff key == c*64 + d)
    probs = torch.zeros(B, A, S, S, device="cuda")
    for c in range(S // 64):
        q2 = qkv.clone()
        v = torch.zeros(B, S, A, 64, device="cuda")
        idx = torch.arange(64, device="cuda")
        v[:, c * 64 + idx, :, idx] = 1.0
        q2[:, 2 * H:] = v.view(B * S, H).to(bf)
        ctx, _ = k.attn_fwd(q2, None, B, S, A, dropout_p=p, seed=seed, dropout_stream=stream)
        probs[:, :, :, c * 64:(c + 1) * 64] = ctx.float().view(B, S, A, 64).permute(0, 2, 1, 3)
    x = qkv.float().view(B, S, 3, A, 64)
    q, kk = x[:, :, 0].permute(0, 2, 1, 3), x[:, :, 1].permute(0, 2, 1, 3)
    pr = torch.softmax(q @ kk.transpose(-1, -2) / 8, -1)
    valid = (pr > 1e-4).cpu().numpy()                     # P~ of a kept element cannot round to zero there
    assert valid.mean() > 0.5, valid.mean()
    got = (probs > 0).cpu().numpy()
    want = reference_keep(B, S, A, p, seed, stream)
    assert 0.88 < want.mean() < 0.92, want.mean()
    bad = np.argwhere(valid & (got != want))
    assert bad.shape[0] == 0, f"{bad.shape[0]} keep bits differ, first (b, h, q, key): {bad[:8].tolist()}"


def test_backward_bitwise_reproducible():
    from deeplearningexamples_b200 import kernels as k
    B, S, A, p = 2, 512, 16, 0.1
    H = A * 64
    g = torch.Generator(device="cuda").manual_seed(8)
    qkv = torch.randn(B * S, 3 * H, generator=g, device="cuda").to(bf)
    dctx = torch.randn(B * S, H, generator=g, device="cuda").to(bf)
    keep = (torch.arange(S, device="cuda").unsqueeze(0) < torch.tensor([S, 300], device="cuda").unsqueeze(1)).float()
    mask = (1.0 - keep) * -10000.0
    ctx, lse = k.attn_fwd(qkv, mask, B, S, A, dropout_p=p, seed=99, dropout_stream=2)
    runs = []
    for _ in range(2):
        dbias = torch.zeros(3 * H, device="cuda")
        dqkv = k.attn_bwd(qkv, mask, ctx, dctx, lse, B, S, A, dropout_p=p, seed=99, dropout_stream=2, dbias=dbias)
        runs.append((dqkv, dbias))
    assert torch.equal(runs[0][0], runs[1][0])
    # the bias gradient is summed across CTAs by fp32 atomics, so only its summation order may differ between calls
    torch.testing.assert_close(runs[0][1], runs[1][1], rtol=1e-5, atol=1e-4)
