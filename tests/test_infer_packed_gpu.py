"""GPU: padding-free inference.  The variable-length attention kernel against an fp32 restatement and, bit for bit, against the
padded kernel; the GELU GEMM without its pre-activation store; and BertModel.remove_padding(True) against the padded forward and
the CPU oracle."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu
bf = torch.bfloat16
LENS = [1, 63, 64, 65, 127, 128, 129, 200, 0, 511, 512]
SENTINEL = -12352.0                       # exactly representable in bf16


def _k():
    from deeplearningexamples_b200 import kernels, _lib
    return kernels, _lib


def _cu(lens):
    cu = [0]
    for n in lens:
        cu.append(cu[-1] + n)
    return torch.tensor(cu, dtype=torch.int32, device="cuda")


def _ref_seq(qkv_rows, A):
    """fp32 softmax(q k^T / 8) v of one sequence's rows [n, 3H] (no mask)."""
    n = qkv_rows.shape[0]
    x = qkv_rows.float().view(n, 3, A, 64)
    q, k, v = (x[:, i].permute(1, 0, 2) for i in range(3))                  # [A, n, 64]
    p = torch.softmax(q @ k.transpose(-1, -2) / math.sqrt(64), dim=-1)
    return (p @ v).permute(1, 0, 2).reshape(n, A * 64)


@pytest.mark.parametrize("A", [1, 16])
def test_varlen_attention_vs_fp32(A):
    k, _ = _k()
    H, extra = A * 64, 40
    T = sum(LENS)
    g = torch.Generator(device="cuda").manual_seed(100 + A)
    qkv = torch.randn(T + extra, 3 * H, generator=g, device="cuda").to(bf)   # the last `extra` rows belong to no sequence
    out = torch.full((T + extra, H), SENTINEL, device="cuda", dtype=bf)
    ctx = k.attn_fwd_varlen(qkv, _cu(LENS), len(LENS), max(LENS), A, out=out)
    assert ctx.data_ptr() == out.data_ptr()
    r0 = 0
    for n in LENS:
        if n:
            torch.testing.assert_close(ctx[r0:r0 + n].float(), _ref_seq(qkv[r0:r0 + n], A), rtol=2e-2, atol=2e-2)
        r0 += n
    assert bool((ctx[T:] == SENTINEL).all()), "a row outside every sequence was written"


def test_varlen_attention_clamps_lengths_to_max_seqlen():
    k, _ = _k()
    A, n, max_s = 2, 300, 256
    g = torch.Generator(device="cuda").manual_seed(7)
    qkv = torch.randn(n, 3 * A * 64, generator=g, device="cuda").to(bf)
    out = torch.full((n, A * 64), SENTINEL, device="cuda", dtype=bf)
    k.attn_fwd_varlen(qkv, _cu([n]), 1, max_s, A, out=out)
    torch.testing.assert_close(out[:max_s].float(), _ref_seq(qkv[:max_s], A), rtol=2e-2, atol=2e-2)
    assert bool((out[max_s:] == SENTINEL).all())


@pytest.mark.parametrize("A", [1, 16])
def test_varlen_attention_bitwise_equals_padded(A):
    """Valid rows of the padded kernel under a -10000 mask, with junk in the padding, equal the packed kernel's bit for bit: the
    padded kernel's extra terms are exact zeros (ex2 of about -14427 flushes to 0; al = ex2(0) = 1 over fully masked tiles)."""
    k, _ = _k()
    H, S, B = A * 64, 512, len(LENS)
    g = torch.Generator(device="cuda").manual_seed(200 + A)
    qkv = torch.randn(sum(LENS), 3 * H, generator=g, device="cuda").to(bf)
    ctx = k.attn_fwd_varlen(qkv, _cu(LENS), B, S, A)
    pad = (torch.randn(B * S, 3 * H, generator=g, device="cuda") * 3.0).to(bf)
    keep = torch.zeros(B, S, device="cuda")
    r0 = 0
    for b, n in enumerate(LENS):
        pad[b * S:b * S + n] = qkv[r0:r0 + n]
        keep[b, :n] = 1.0
        r0 += n
    ctx_pad, _ = k.attn_fwd(pad, (1.0 - keep) * -10000.0, B, S, A)
    assert torch.equal(ctx_pad[keep.view(-1) != 0], ctx)


@pytest.mark.parametrize("shape", [(40, 264, 72), (1096, 800, 200), (8320, 1024, 128)], ids=lambda s: f"{s[0]}x{s[1]}x{s[2]}")
@pytest.mark.parametrize("bn", [128, 256])
@pytest.mark.parametrize("layout", ["kk", "kmn", "mnmn", "mnk"])
def test_gelu_gemm_without_preactivation_store(layout, bn, shape):
    k, L = _k()
    M, N, K = shape
    g = torch.Generator().manual_seed(M + N + K + bn)
    a_mn, b_mn = layout.startswith("mn"), layout.endswith("mn")
    a = torch.randn((K, M) if a_mn else (M, K), generator=g).to(bf).cuda()
    b = (torch.randn((K, N) if b_mn else (N, K), generator=g) * 0.1).to(bf).cuda()
    bias = torch.randn(N, generator=g).to(bf).cuda()
    kw = dict(a_layout=L.LAYOUT_MN if a_mn else L.LAYOUT_K, b_layout=L.LAYOUT_MN if b_mn else L.LAYOUT_K, tile_n=bn if bn == 128 else 0,
              bias=bias, epilogue=L.EPI_BIAS_GELU)
    y, u = k.gemm(a, b, **kw)
    y_only, none = k.gemm(a, b, out2=False, **kw)
    assert none is None and torch.equal(y, y_only)


# ------------------------------------------------------------------------------------------------------------------------------
# model
# ------------------------------------------------------------------------------------------------------------------------------
SMALL = dict(hidden_size=256, num_hidden_layers=2, num_attention_heads=4, intermediate_size=1024, vocab_size=1024,
             max_position_embeddings=512, type_vocab_size=2, hidden_act="gelu", initializer_range=0.02)
LARGE2 = dict(SMALL, hidden_size=1024, num_attention_heads=16, intermediate_size=4096, vocab_size=2048)


def _models(cfg, seed):
    from deeplearningexamples_b200 import modeling
    from oracle import bert_oracle as O
    sd = O.bf16_representable_params(cfg, seed=seed)
    c = modeling.BertConfig.from_dict({**cfg, "hidden_dropout_prob": 0.1, "attention_probs_dropout_prob": 0.1})
    pre = modeling.BertForPreTraining(c)
    full = dict(sd, **{"cls.predictions.decoder.weight": sd["bert.embeddings.word_embeddings.weight"]})
    missing, unexpected = pre.load_state_dict(full, strict=False)
    assert not missing and not unexpected, (missing, unexpected)
    torch.manual_seed(seed)
    qa = modeling.BertForQuestionAnswering(c)
    qa.load_state_dict(sd, strict=False)
    qa.qa_outputs.weight.data.copy_(torch.randn(2, cfg["hidden_size"]) * 0.05)
    return sd, pre.cuda().to(bf).eval(), qa.cuda().to(bf).eval()


def _batch(B, S, vocab, seed, lens, holes_row=None, empty_row=None):
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(0, vocab, (B, S), generator=g)
    ids[:, 0] = 101
    tt = torch.zeros(B, S, dtype=torch.long)
    tt[:, S // 2:] = 1
    am = (torch.arange(S).unsqueeze(0) < torch.tensor(lens).unsqueeze(1)).long()
    if holes_row is not None:                      # a mask that is not a prefix: position 0 kept, holes everywhere else
        am[holes_row] = (torch.rand(S, generator=g) < 0.6).long()
        am[holes_row, 0] = 1
    if empty_row is not None:
        am[empty_row] = 0
    return ids, tt, am


def _run(model, ids, tt, am, remove_padding):
    model.remove_padding(remove_padding)
    try:
        with torch.no_grad():
            return model(ids.cuda(), tt.cuda(), am.cuda())
    finally:
        model.remove_padding(False)


def _rel(got, want):
    return ((got.float() - want.float()).abs().max() / want.float().abs().max().clamp_min(1e-12)).item()


def _rel_l2(got, want):
    return ((got.float() - want.float()).norm() / want.float().norm().clamp_min(1e-12)).item()


@pytest.mark.parametrize("cfg,B,S,lens", [(SMALL, 6, 128, [128, 1, 77, 100, 0, 0]), (LARGE2, 4, 512, [512, 129, 0, 0])],
                         ids=["small", "large-width-2-layers"])
def test_model_packed_equals_padded(cfg, B, S, lens):
    from oracle import bert_oracle as O
    sd, pre, qa = _models(cfg, seed=41)
    holes, empty = B - 2, B - 1                     # the last two rows: a non-prefix mask and an all-zero mask
    ids, tt, am = _batch(B, S, cfg["vocab_size"], seed=5, lens=lens, holes_row=holes, empty_row=empty)
    (enc_pad,), pooled_pad = _run(pre.bert, ids, tt, am, False)
    (enc_pk,), pooled_pk = _run(pre.bert, ids, tt, am, True)
    keep = am.cuda() != 0
    right = torch.ones(B, dtype=torch.bool, device="cuda")
    right[holes] = right[empty] = False
    # right-padded rows: bit for bit (row results of the GEMM and LayerNorm do not depend on the other rows; attention by the
    # exact-zero argument); masked positions: exactly zero
    rk = keep & right.unsqueeze(1)
    assert torch.equal(enc_pk[rk], enc_pad[rk])
    assert torch.count_nonzero(enc_pk[~keep]) == 0
    assert torch.equal(pooled_pk[right], pooled_pad[right])
    # the non-prefix row: its kept keys fall into different 64-key tiles than in the padded batch, so the online softmax rescales
    # and the MMA's k-groups differ -- equal within bf16 rounding, not bitwise
    hk = keep[holes]
    assert _rel_l2(enc_pk[holes][hk], enc_pad[holes][hk]) < 1e-2
    # CPU oracle on the valid positions of every non-empty row
    with torch.no_grad():
        seq_ref, _ = O.bert_model(sd, cfg, ids, tt, am)
    valid = (am != 0) & (torch.arange(B) != empty).unsqueeze(1)
    got = enc_pk.cpu()[valid]
    assert _rel_l2(got, seq_ref[valid]) < 1e-2 and _rel(got, seq_ref[valid]) < 3e-2
    # span head: logits at valid positions equal (right-padded rows)
    start_pad, end_pad = _run(qa, ids, tt, am, False)
    start_pk, end_pk = _run(qa, ids, tt, am, True)
    assert torch.equal(start_pk[rk], start_pad[rk]) and torch.equal(end_pk[rk], end_pad[rk])


def test_model_output_all_encoded_layers_packed():
    from deeplearningexamples_b200 import modeling
    cfg = dict(SMALL, output_all_encoded_layers=True)
    _, pre, _ = _models(cfg, seed=43)
    B, S = 3, 128
    ids, tt, am = _batch(B, S, cfg["vocab_size"], seed=6, lens=[128, 40, 90])
    layers_pad, _ = _run(pre.bert, ids, tt, am, False)
    layers_pk, _ = _run(pre.bert, ids, tt, am, True)
    assert len(layers_pk) == len(layers_pad) == cfg["num_hidden_layers"]
    keep = (am.cuda() != 0).t()                     # layers come as (seq, bsz, hidden), as on the padded path
    for a, b in zip(layers_pk, layers_pad):
        assert a.shape == b.shape == (S, B, cfg["hidden_size"])
        assert torch.equal(a[keep], b[keep]) and torch.count_nonzero(a[~keep]) == 0


def test_full_mask_batch_takes_the_padded_path(monkeypatch):
    k, L = _k()
    sd, pre, _ = _models(SMALL, seed=44)
    ids, tt, am = _batch(3, 256, SMALL["vocab_size"], seed=7, lens=[256, 256, 256])
    (enc_off,), pooled_off = _run(pre.bert, ids, tt, am, False)

    def _no_varlen(*a, **kw):
        raise AssertionError("a full-mask batch must not take the packed route")
    monkeypatch.setattr(k, "attn_fwd_varlen", _no_varlen)
    (enc_on,), pooled_on = _run(pre.bert, ids, tt, am, True)
    assert torch.equal(enc_on, enc_off) and torch.equal(pooled_on, pooled_off)


@pytest.mark.parametrize("S", [200, 64])
def test_any_sequence_length_with_remove_padding(S):
    from oracle import bert_oracle as O
    k, L = _k()
    sd, pre, _ = _models(SMALL, seed=45)
    for lens in ([S, S // 2, 1], [S, S, S]):
        ids, tt, am = _batch(3, S, SMALL["vocab_size"], seed=8, lens=lens)
        (enc,), pooled = _run(pre.bert, ids, tt, am, True)
        with torch.no_grad():
            seq_ref, _ = O.bert_model(sd, SMALL, ids, tt, am)
        valid = am != 0
        got = enc.cpu()[valid]
        assert _rel_l2(got, seq_ref[valid]) < 1e-2 and _rel(got, seq_ref[valid]) < 3e-2, lens
        assert torch.count_nonzero(enc[~valid.cuda()]) == 0
        with pytest.raises(L.DleError):
            _run(pre.bert, ids, tt, am, False)                  # the padded attention still takes S % 128 == 0 only
