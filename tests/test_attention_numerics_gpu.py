"""The fused attention kernels against fp64 (test_attention_numerics_cpu.py holds the references, yardsticks and bars, and shows on the
CPU that a correct kernel clears the bars and subtly wrong ones do not): the padded forward and backward over the input families at
every S and at tile-edge masks, the seq-first layout bit for bit against batch-first, exact invariants, and the packed training
kernels.  The largest score seen per family and bar is reported at the end of the module."""
import collections

import pytest
import torch

from test_attention_numerics_cpu import (BARS, FAMILIES, HD, attention_ref64, backward_yardstick, bwd_ratios, edge_lens, elem_floor,
                                         family_qkv, forward_scores, keep_mask, lens_mask, over_bars, rand_dctx)

pytestmark = pytest.mark.gpu
DEV = "cuda"
P_DROP, STREAM = 0.1, 5
_WORST = collections.defaultdict(dict)


def _k():
    from deeplearningexamples_b200 import kernels
    return kernels


@pytest.fixture(scope="module", autouse=True)
def _report(request):
    yield
    if _WORST:
        lines = ["", "fused attention on the GPU vs fp64: largest score per family (bars: " +
                 ", ".join(f"{k} <= {v:g}" for k, v in BARS.items()) + ")",
                 f"{'family':<22}" + "".join(f"{k:>10}" for k in BARS)]
        for fam in sorted(_WORST):
            lines.append(f"{fam:<22}" + "".join(f"{_WORST[fam].get(k, float('nan')):10.3f}" for k in BARS))
        capman = request.config.pluginmanager.getplugin("capturemanager")
        with capman.global_and_fixture_disabled():
            print("\n".join(lines))


def _record(label, sc):
    for key, v in sc.items():
        _WORST[label][key] = max(_WORST[label].get(key, 0.0), v)
    assert over_bars(sc) == [], (label, sc)


def _run_padded(qkv, mask, dctx, B, S, A, p, seed, seq_first=False, dbias=None):
    k = _k()
    ctx, lse = k.attn_fwd(qkv, mask, B, S, A, dropout_p=p, seed=seed, dropout_stream=STREAM, seq_first=seq_first)
    dqkv = k.attn_bwd(qkv, mask, ctx, dctx, lse, B, S, A, dropout_p=p, seed=seed, dropout_stream=STREAM, seq_first=seq_first,
                      dbias=dbias)
    return ctx, lse, dqkv


def _scores_padded(qkv, mask, dctx, B, S, A, p, seed, seq_first=False):
    """the kernels' outputs and their bar scores against fp64"""
    keep = keep_mask(B, S, A, p, seed, STREAM, DEV)
    ctx, lse, dqkv = _run_padded(qkv, mask, dctx, B, S, A, p, seed, seq_first)
    ref_ctx, ref_lse, ref_dqkv = attention_ref64(qkv, mask, B, S, A, seq_first, keep, p, dctx)
    yard = backward_yardstick(qkv, mask, ctx, dctx, ref_lse, B, S, A, seq_first, keep, p)
    sc = forward_scores(ctx, lse, ref_ctx, ref_lse, elem_floor(qkv, mask, B, S, A, seq_first))
    sc.update(bwd_ratios(dqkv, yard, ref_dqkv, A * HD))
    return sc


def _to_seq_first(x, B, S):
    return x.view(B, S, -1).transpose(0, 1).contiguous().view(B * S, -1)


@pytest.mark.parametrize("A", [1, 16])
@pytest.mark.parametrize("S", [128, 256, 384, 512])
@pytest.mark.parametrize("family", FAMILIES)
def test_padded_vs_fp64(family, S, A):
    """an unmasked pair of rows without dropout, and one row per tile-edge length plus an all-padding row under dropout 0.1"""
    seed = 100 * FAMILIES.index(family) + S + A
    qkv = family_qkv(family, 2, S, A, seed=seed, device=DEV)
    _record(family, _scores_padded(qkv, None, rand_dctx(2 * S, A * HD, seed + 1, DEV), 2, S, A, 0.0, seed))
    lens = edge_lens(S)
    B = len(lens)
    qkv = family_qkv(family, B, S, A, lens, seed=seed + 2, device=DEV)
    _record(family, _scores_padded(qkv, lens_mask(lens, S, DEV), rand_dctx(B * S, A * HD, seed + 3, DEV), B, S, A, P_DROP, seed))


@pytest.mark.parametrize("family", FAMILIES)
def test_padded_multi_wave_vs_fp64(family):
    """B=4, A=16, S=512: 256 forward CTAs and 512 backward CTAs per kernel, more than one wave on 132 SMs"""
    B, S, A, seed = 4, 512, 16, 7 + FAMILIES.index(family)
    lens = [S, 511, 129, 64]
    qkv = family_qkv(family, B, S, A, lens, seed=seed, device=DEV)
    _record(family, _scores_padded(qkv, lens_mask(lens, S, DEV), rand_dctx(B * S, A * HD, seed + 1, DEV), B, S, A, P_DROP, seed))


@pytest.mark.parametrize("S", [128, 256, 384, 512])
def test_seq_first_bitwise_equals_batch_first(S):
    """attn_fwd / attn_bwd on the [S, B, *] token order give the bits of the batch-first call on the transposed copy -- ctx, lse,
    dqkv -- with dropout and a ragged mask; at S = 512 the seq-first call is also held to the fp64 bars."""
    B, A, seed = 3, 2, 31 + S
    lens = [S, S // 2 + 1, 63]
    mask = lens_mask(lens, S, DEV)
    qkv = family_qkv("sharp3", B, S, A, lens, seed=seed, device=DEV)
    dctx = rand_dctx(B * S, A * HD, seed + 1, DEV)
    qkv_sf, dctx_sf = _to_seq_first(qkv, B, S), _to_seq_first(dctx, B, S)
    db_bf, db_sf = torch.zeros(3 * A * HD, device=DEV), torch.zeros(3 * A * HD, device=DEV)
    ctx, lse, dqkv = _run_padded(qkv, mask, dctx, B, S, A, P_DROP, seed, dbias=db_bf)
    ctx_sf, lse_sf, dqkv_sf = _run_padded(qkv_sf, mask, dctx_sf, B, S, A, P_DROP, seed, seq_first=True, dbias=db_sf)
    assert torch.equal(ctx_sf, _to_seq_first(ctx, B, S))
    assert torch.equal(lse_sf, lse)
    assert torch.equal(dqkv_sf, _to_seq_first(dqkv, B, S))
    torch.testing.assert_close(db_sf, db_bf, rtol=1e-5, atol=1e-4)          # fp32 atomics: only the summation order differs
    if S == 512:
        _record("seq_first sharp3", _scores_padded(qkv_sf, mask, dctx_sf, B, S, A, P_DROP, seed, seq_first=True))


@pytest.mark.parametrize("S", [128, 512])
def test_lse_bitwise_independent_of_dropout(S):
    """l is summed before the keep mask, so lse with dropout is bitwise lse without"""
    lens = edge_lens(S)
    B, A = len(lens), 4
    qkv = family_qkv("rising", B, S, A, lens, seed=S, device=DEV)
    mask = lens_mask(lens, S, DEV)
    _, lse0 = _k().attn_fwd(qkv, mask, B, S, A)
    _, lse1 = _k().attn_fwd(qkv, mask, B, S, A, dropout_p=P_DROP, seed=3, dropout_stream=STREAM)
    assert torch.equal(lse0, lse1)


@pytest.mark.parametrize("p", [0.0, P_DROP])
@pytest.mark.parametrize("seq_first", [False, True])
def test_exact_zeros(seq_first, p):
    """Query rows whose dctx is zero get a dQ row of exactly 0; keys past a row's length (in a row with at least one valid key) get
    dK and dV rows of exactly 0; every edge length, both token orders.  dbias is the column sum of the stored dqkv, to within the
    rounding of its fp32 sums."""
    S, A = 512, 2
    lens = edge_lens(S)
    B, H = len(lens), A * HD
    qkv = family_qkv("sharp3", B, S, A, lens, seed=41, device=DEV)
    mask = lens_mask(lens, S, DEV)
    dctx = rand_dctx(B * S, H, 42, DEV)
    zero_q = torch.arange(B * S, device=DEV) % 3 == 1
    dctx[zero_q] = 0
    pos = torch.arange(S, device=DEV)
    masked_key = ((pos.unsqueeze(0) >= torch.tensor(lens, device=DEV).unsqueeze(1)) &
                  (torch.tensor(lens, device=DEV) > 0).unsqueeze(1)).view(-1)     # [B*S] batch-first
    if seq_first:
        qkv, dctx, zero_q = _to_seq_first(qkv, B, S), _to_seq_first(dctx, B, S), _to_seq_first(zero_q.view(-1, 1), B, S).view(-1)
        masked_key = _to_seq_first(masked_key.view(-1, 1), B, S).view(-1)
    dbias = torch.zeros(3 * H, device=DEV)
    _, _, dqkv = _run_padded(qkv, mask, dctx, B, S, A, p, 43, seq_first, dbias=dbias)
    assert torch.count_nonzero(dqkv[zero_q, :H]) == 0
    assert torch.count_nonzero(dqkv[masked_key, H:]) == 0
    assert torch.count_nonzero(dqkv[~masked_key, H:]) > 0
    # each column is B*S/16 atomic adds of warp partials (16-row sums): worst-case fp32 error (n + 16) * 2^-24 * sum |x|
    col = dqkv.double()
    bound = (B * S / 16 + 16) * 2.0 ** -24 * col.abs().sum(0)
    assert ((dbias.double() - col.sum(0)).abs() <= bound).all()


VARLEN_LENS = [1, 63, 64, 65, 127, 129, 0, 511, 512]


@pytest.mark.parametrize("p", [0.0, P_DROP])
@pytest.mark.parametrize("family", ["sharp3", "sharp5", "spike_late", "rising"])
def test_varlen_train_vs_fp64(family, p):
    """attn_fwd_varlen_train / attn_bwd_varlen (their own copy of the online-softmax loop) on packed sequences of tile-edge lengths,
    each sequence against attention_ref64 with the keep bits keyed at drop_stride = 512.  Sequences of one token have exactly zero
    dq / dk, so the backward bars apply to the others one by one and to all of them together."""
    k = _k()
    A, stride, seed = 4, 512, 61 + FAMILIES.index(family)
    H, B = A * HD, len(VARLEN_LENS)
    cu = [0]
    for n in VARLEN_LENS:
        cu.append(cu[-1] + n)
    T = cu[-1]
    qkv = torch.cat([family_qkv(family, 1, n, A, seed=seed + i, device=DEV) for i, n in enumerate(VARLEN_LENS) if n > 0])
    dctx = rand_dctx(T, H, seed + 100, DEV)
    cu_t = torch.tensor(cu, dtype=torch.int32, device=DEV)
    ctx, lse = k.attn_fwd_varlen_train(qkv, cu_t, B, max(VARLEN_LENS), A, stride, dropout_p=p, seed=seed, dropout_stream=STREAM)
    dqkv = k.attn_bwd_varlen(qkv, cu_t, ctx, dctx, lse, B, max(VARLEN_LENS), A, stride, dropout_p=p, seed=seed, dropout_stream=STREAM)
    keep = keep_mask(B, stride, A, p, seed, STREAM, DEV)
    ref_ctx, ref_lse = torch.empty(T, H, dtype=torch.float64, device=DEV), torch.empty(A, T, dtype=torch.float64, device=DEV)
    ref_dqkv, yard = torch.empty(T, 3 * H, dtype=torch.float64, device=DEV), torch.empty(T, 3 * H, dtype=torch.float64, device=DEV)
    floor = torch.empty(T, H, dtype=torch.float64, device=DEV)
    label = f"varlen {family}"
    for b, n in enumerate(VARLEN_LENS):
        if n == 0:
            continue
        r = slice(cu[b], cu[b + 1])
        kb = keep[b:b + 1, :, :n, :n] if keep is not None else None
        c, l, d = attention_ref64(qkv[r], None, 1, n, A, keep=kb, p=p, dctx=dctx[r])
        ref_ctx[r], ref_lse[:, r], ref_dqkv[r] = c, l[0], d
        yard[r] = backward_yardstick(qkv[r], None, ctx[r], dctx[r], l, 1, n, A, keep=kb, p=p)
        floor[r] = elem_floor(qkv[r], None, 1, n, A)
        sc = forward_scores(ctx[r], lse[:, r].unsqueeze(0), c, l, floor[r])
        if n > 1:
            sc.update(bwd_ratios(dqkv[r], yard[r], d, H))
        _record(label, sc)
    sc = forward_scores(ctx, lse, ref_ctx, ref_lse, floor)
    sc.update(bwd_ratios(dqkv, yard, ref_dqkv, H))
    _record(label, sc)
