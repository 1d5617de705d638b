"""GPU: padding-free training.  The variable-length attention forward (dropout, lse) and backward against fp32 restatements and, bit
for bit, against the padded kernels; ops.BertLayerPackedFn against ops.BertLayerFn; BertForPreTraining with
remove_padding(True, training=True) against the padded route and the CPU oracle; and a few LAMB steps on the route."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu
bf = torch.bfloat16
LENS = [1, 63, 64, 65, 200, 0, 511, 512, 128, 0]
SENTINEL = -12352.0                       # exactly representable in bf16


def _k():
    from deeplearningexamples_b200 import kernels
    return kernels


def _cu(lens):
    cu = [0]
    for n in lens:
        cu.append(cu[-1] + n)
    return torch.tensor(cu, dtype=torch.int32, device="cuda")


def _rel_l2(got, want):
    return ((got.float() - want.float()).norm() / want.float().norm().clamp_min(1e-12)).item()


def _cos(got, want):
    return torch.nn.functional.cosine_similarity(got.float().flatten(), want.float().flatten(), dim=0).item()


def _ref_seq(qkv_rows, A, dctx_rows=None):
    """fp32 restatement of one sequence [n, 3H]: (ctx [n, H], lse [A, n]) and, given dctx, d(qkv) [n, 3H] of sum(ctx * dctx)."""
    n = qkv_rows.shape[0]
    x = qkv_rows.float().clone().requires_grad_(dctx_rows is not None)
    q, k, v = (x.view(n, 3, A, 64)[:, i].permute(1, 0, 2) for i in range(3))     # [A, n, 64]
    s = q @ k.transpose(-1, -2) / math.sqrt(64)
    ctx = (torch.softmax(s, dim=-1) @ v).permute(1, 0, 2).reshape(n, A * 64)
    lse = torch.logsumexp(s, dim=-1)
    if dctx_rows is None:
        return ctx.detach(), lse.detach(), None
    (ctx * dctx_rows.float()).sum().backward()
    return ctx.detach(), lse.detach(), x.grad


def _padded(qkv, lens, S, A, g):
    """The packed rows laid out on a right-padded [B, S] grid with junk in the padding, and the -10000 additive mask."""
    B = len(lens)
    pad = (torch.randn(B * S, qkv.shape[1], generator=g, device="cuda") * 3.0).to(bf)
    keep = torch.zeros(B, S, device="cuda")
    r0 = 0
    for b, n in enumerate(lens):
        pad[b * S:b * S + n] = qkv[r0:r0 + n]
        keep[b, :n] = 1.0
        r0 += n
    return pad, keep, (1.0 - keep) * -10000.0


# ------------------------------------------------------------------------------------------------------------------------------
# kernels
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("A", [1, 16])
def test_forward_without_dropout_equals_inference_kernel_and_fp32_lse(A):
    k = _k()
    H, T, B = A * 64, sum(LENS), len(LENS)
    g = torch.Generator(device="cuda").manual_seed(300 + A)
    qkv = torch.randn(T, 3 * H, generator=g, device="cuda").to(bf)
    cu = _cu(LENS)
    ctx, lse = k.attn_fwd_varlen_train(qkv, cu, B, 512, A, 512, dropout_p=0.0, seed=11, dropout_stream=5)
    assert lse.shape == (A, T) and lse.dtype == torch.float32
    assert torch.equal(ctx, k.attn_fwd_varlen(qkv, cu, B, 512, A))
    r0 = 0
    for n in LENS:
        if n:
            _, lse_ref, _ = _ref_seq(qkv[r0:r0 + n], A)
            torch.testing.assert_close(lse[:, r0:r0 + n], lse_ref, rtol=1e-4, atol=2e-4)
        r0 += n


@pytest.mark.parametrize("A", [1, 16])
def test_forward_with_dropout_bitwise_equals_padded_kernel(A):
    k = _k()
    H, T, B, S = A * 64, sum(LENS), len(LENS), 512
    g = torch.Generator(device="cuda").manual_seed(400 + A)
    qkv = torch.randn(T, 3 * H, generator=g, device="cuda").to(bf)
    ctx, lse = k.attn_fwd_varlen_train(qkv, _cu(LENS), B, max(LENS), A, S, dropout_p=0.1, seed=12345, dropout_stream=9)
    pad, keep, mask = _padded(qkv, LENS, S, A, g)
    ctx_pad, lse_pad = k.attn_fwd(pad, mask, B, S, A, dropout_p=0.1, seed=12345, dropout_stream=9)
    assert torch.equal(ctx_pad[keep.view(-1) != 0], ctx)
    lse_pad_valid = lse_pad.permute(1, 0, 2)[:, keep != 0]               # [A, T] in packed order
    assert torch.equal(lse_pad_valid, lse)
    # dropout is really on: the same call without it differs
    ctx0, _ = k.attn_fwd_varlen_train(qkv, _cu(LENS), B, max(LENS), A, S, dropout_p=0.0)
    assert not torch.equal(ctx0, ctx)


@pytest.mark.parametrize("A", [1, 16])
def test_backward_vs_fp32(A):
    k = _k()
    H, T, B, extra = A * 64, sum(LENS), len(LENS), 40
    g = torch.Generator(device="cuda").manual_seed(500 + A)
    qkv = torch.randn(T + extra, 3 * H, generator=g, device="cuda").to(bf)      # the last `extra` rows belong to no sequence
    dctx = torch.randn(T + extra, H, generator=g, device="cuda").to(bf)
    cu = _cu(LENS)
    ctx, lse = k.attn_fwd_varlen_train(qkv, cu, B, 512, A, 512)
    out = torch.full((T + extra, 3 * H), SENTINEL, device="cuda", dtype=bf)
    dbias = torch.zeros(3 * H, device="cuda")
    dqkv = k.attn_bwd_varlen(qkv, cu, ctx, dctx, lse, B, 512, A, 512, dbias=dbias, out=out)
    assert dqkv.data_ptr() == out.data_ptr()
    assert bool((dqkv[T:] == SENTINEL).all()), "a row outside every sequence was written"
    assert bool(torch.isfinite(dqkv[:T].float()).all()) and bool(torch.isfinite(dbias).all())
    refs, r0 = [], 0
    for n in LENS:
        if n:
            _, _, d_ref = _ref_seq(qkv[r0:r0 + n], A, dctx[r0:r0 + n])
            refs.append(d_ref)
            got = dqkv[r0:r0 + n]
            assert _rel_l2(got, d_ref) < 2e-2, (n, _rel_l2(got, d_ref))
            for part in range(3):                                          # dq, dk and dv each
                w = d_ref[:, part * H:(part + 1) * H]
                if w.norm() > 1e-3:
                    assert _rel_l2(got[:, part * H:(part + 1) * H], w) < 3e-2, (n, part)
        r0 += n
    db_ref = torch.cat(refs).sum(0)
    assert _rel_l2(dbias, db_ref) < 2e-2


@pytest.mark.parametrize("A", [1, 16])
def test_backward_with_dropout_bitwise_equals_padded_kernel(A):
    k = _k()
    H, T, B, S = A * 64, sum(LENS), len(LENS), 512
    g = torch.Generator(device="cuda").manual_seed(600 + A)
    qkv = torch.randn(T, 3 * H, generator=g, device="cuda").to(bf)
    dctx = torch.randn(T, H, generator=g, device="cuda").to(bf)
    cu = _cu(LENS)
    kw = dict(dropout_p=0.1, seed=777, dropout_stream=4)
    ctx, lse = k.attn_fwd_varlen_train(qkv, cu, B, max(LENS), A, S, **kw)
    db = torch.zeros(3 * H, device="cuda")
    dqkv = k.attn_bwd_varlen(qkv, cu, ctx, dctx, lse, B, max(LENS), A, S, dbias=db, **kw)
    pad, keep, mask = _padded(qkv, LENS, S, A, g)
    sel = keep.view(-1) != 0
    ctx_pad, lse_pad = k.attn_fwd(pad, mask, B, S, A, **kw)
    dctx_pad = torch.zeros(B * S, H, device="cuda", dtype=bf)
    dctx_pad[sel] = dctx                                                   # dO = 0 on padded rows
    db_pad = torch.zeros(3 * H, device="cuda")
    dqkv_pad = k.attn_bwd(pad, mask, ctx_pad, dctx_pad, lse_pad, B, S, A, dbias=db_pad, **kw)
    assert torch.equal(dqkv_pad[sel], dqkv)
    torch.testing.assert_close(db, db_pad, rtol=1e-4, atol=1e-4 * db_pad.abs().max().item())
    again = k.attn_bwd_varlen(qkv, cu, ctx, dctx, lse, B, max(LENS), A, S, **kw)
    assert torch.equal(again, dqkv)


def test_backward_of_all_empty_sequences_writes_nothing():
    k = _k()
    A, T = 2, 64
    qkv = torch.randn(T, 3 * A * 64, device="cuda").to(bf)
    cu = torch.zeros(4, dtype=torch.int32, device="cuda")                  # three sequences of length 0
    ctx, lse = k.attn_fwd_varlen_train(qkv, cu, 3, 64, A, 64, dropout_p=0.1, seed=3)
    out = torch.full_like(qkv, SENTINEL)
    db = torch.zeros(3 * A * 64, device="cuda")
    k.attn_bwd_varlen(qkv, cu, ctx, torch.zeros_like(ctx), lse, 3, 64, A, 64, dropout_p=0.1, seed=3, dbias=db, out=out)
    assert bool((out == SENTINEL).all()) and torch.count_nonzero(db) == 0


# ------------------------------------------------------------------------------------------------------------------------------
# autograd node and model
# ------------------------------------------------------------------------------------------------------------------------------
SMALL = dict(hidden_size=256, num_hidden_layers=2, num_attention_heads=4, intermediate_size=1024, vocab_size=1024,
             max_position_embeddings=512, type_vocab_size=2, hidden_act="gelu", initializer_range=0.02)


def _config(cfg, p_hidden, p_attn):
    from deeplearningexamples_b200 import modeling
    return modeling.BertConfig.from_dict({**cfg, "hidden_dropout_prob": p_hidden, "attention_probs_dropout_prob": p_attn})


def _pack_index(keep):
    lens = keep.sum(1).to(torch.int32)
    cu = torch.zeros(keep.shape[0] + 1, dtype=torch.int32, device="cuda")
    torch.cumsum(lens, 0, dtype=torch.int32, out=cu[1:])
    return torch.nonzero(keep.reshape(-1)).squeeze(-1), cu, int(lens.max())


def _grads(module):
    out = {n: p.grad.detach().clone() for n, p in module.named_parameters() if p.grad is not None}
    module.zero_grad(set_to_none=True)
    return out


def _assert_param_grads_agree(got, want, cos_min, rel_max):
    assert got.keys() == want.keys()
    for n in want:
        if want[n].float().norm() > 0:
            assert _cos(got[n], want[n]) > cos_min and _rel_l2(got[n], want[n]) < rel_max, (n, _cos(got[n], want[n]),
                                                                                            _rel_l2(got[n], want[n]))


def test_packed_layer_node_equals_padded_layer_node():
    from deeplearningexamples_b200 import modeling, ops
    torch.manual_seed(21)
    layer = modeling.BertLayer(_config(SMALL, 0.0, 0.1)).cuda().to(bf).train()
    B, S, H = 4, 256, SMALL["hidden_size"]
    lens = torch.tensor([256, 200, 1, 65], device="cuda")
    keep = torch.arange(S, device="cuda").unsqueeze(0) < lens.unsqueeze(1)
    g = torch.Generator(device="cuda").manual_seed(22)
    x0 = torch.randn(B, S, H, generator=g, device="cuda").to(bf)
    dy = torch.randn(B, S, H, generator=g, device="cuda").to(bf) * keep.unsqueeze(-1)
    mask = ((~keep).float() * -10000.0).view(B, 1, 1, S)

    ops.manual_seed(5)
    x = x0.clone().requires_grad_()
    y_pad = layer(x.transpose(0, 1), mask).transpose(0, 1)
    y_pad.backward(dy)
    dx_pad, g_pad = x.grad.clone(), _grads(layer)

    ops.manual_seed(5)
    idx, cu, max_len = _pack_index(keep)
    x = x0.clone().requires_grad_()
    xp = ops.GatherRowsFn.apply(x.view(B * S, H), idx)
    y_pk = ops.ScatterRowsFn.apply(layer.forward_packed(xp, cu, max_len, S), idx, B * S).view(B, S, H)
    y_pk.backward(dy)
    dx_pk, g_pk = x.grad.clone(), _grads(layer)

    assert torch.equal(y_pk[keep], y_pad[keep]) and torch.count_nonzero(y_pk[~keep]) == 0
    assert torch.equal(dx_pk[keep], dx_pad[keep]) and torch.count_nonzero(dx_pk[~keep]) == 0
    _assert_param_grads_agree(g_pk, g_pad, 0.9999, 1e-2)


def _batch(B, S, vocab, lens, seed, holes_row=None, n_labels=8):
    """Right-padded rows of the given lengths (a non-prefix mask on holes_row, position 0 kept), MLM labels on kept positions only."""
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(0, vocab, (B, S), generator=g)
    ids[:, 0] = 101
    tt = torch.zeros(B, S, dtype=torch.long)
    tt[:, S // 2:] = 1
    am = (torch.arange(S).unsqueeze(0) < torch.tensor(lens).unsqueeze(1)).long()
    if holes_row is not None:
        am[holes_row] = (torch.rand(S, generator=g) < 0.6).long()
        am[holes_row, 0] = 1
    labels = torch.full((B, S), -1, dtype=torch.long)
    for b in range(B):
        kept = torch.nonzero(am[b]).squeeze(-1)
        pos = kept[torch.randperm(kept.numel(), generator=g)[:n_labels]]
        labels[b, pos] = torch.randint(0, vocab, (pos.numel(),), generator=g)
    nsl = torch.randint(0, 2, (B,), generator=g)
    return {"input_ids": ids, "token_type_ids": tt, "attention_mask": am, "labels": labels, "next_sentence_labels": nsl}


def _pretraining_model(cfg, p_hidden, p_attn, sd):
    from deeplearningexamples_b200 import modeling
    m = modeling.BertForPreTraining(_config(cfg, p_hidden, p_attn), sequence_output_is_dense=True)
    full = dict(sd, **{"cls.predictions.decoder.weight": sd["bert.embeddings.word_embeddings.weight"]})
    missing, unexpected = m.load_state_dict(full, strict=False)
    assert not missing and not unexpected, (missing, unexpected)
    return m.cuda().to(bf).train()


def _step(model, batch, seed):
    """One forward + backward in train mode: (scores, nsp, loss, gradient at the embedding output, parameter gradients)."""
    from deeplearningexamples_b200 import ops, training
    emb = []

    def hook(mod, inp, out):
        out.retain_grad()
        emb.append(out)
    h = model.bert.embeddings.register_forward_hook(hook)
    try:
        ops.manual_seed(seed)
        b = {k: v.cuda() for k, v in batch.items()}
        scores, nsp = model(b["input_ids"], b["token_type_ids"], b["attention_mask"], b["labels"])
        crit = training.BertPretrainingCriterion(model.config.vocab_size, sequence_output_is_dense=True)
        loss = crit(scores, nsp, b["labels"], b["next_sentence_labels"])
        loss.backward()
    finally:
        h.remove()
    return scores.detach(), nsp.detach(), loss.detach(), emb[0].grad.detach().clone(), _grads(model)


def test_pretraining_model_packed_equals_padded():
    from oracle import bert_oracle as O
    sd = O.bf16_representable_params(SMALL, seed=51)
    model = _pretraining_model(SMALL, 0.0, 0.1, sd)
    B, S = 4, 128
    batch = _batch(B, S, SMALL["vocab_size"], [128, 77, 1, 100], seed=52)
    model.remove_padding(False)
    s_pad, n_pad, l_pad, e_pad, g_pad = _step(model, batch, seed=9)
    model.remove_padding(True, training=True)
    s_pk, n_pk, l_pk, e_pk, g_pk = _step(model, batch, seed=9)
    model.remove_padding(False)
    assert torch.equal(s_pk, s_pad) and torch.equal(n_pk, n_pad) and torch.equal(l_pk, l_pad)
    keep = batch["attention_mask"].cuda() != 0
    assert torch.equal(e_pk[keep], e_pad[keep]) and torch.count_nonzero(e_pk[~keep]) == 0
    _assert_param_grads_agree(g_pk, g_pad, 0.9999, 1e-2)


@pytest.mark.parametrize("S,lens,holes_row", [(128, [128, 90, 128], 2), (200, [200, 37, 150], None)], ids=["holes", "S200"])
def test_pretraining_gradients_vs_cpu_oracle(S, lens, holes_row):
    from oracle import bert_oracle as O
    sd = O.bf16_representable_params(SMALL, seed=61)
    model = _pretraining_model(SMALL, 0.0, 0.0, sd)
    model.remove_padding(True, training=True)
    batch = _batch(len(lens), S, SMALL["vocab_size"], lens, seed=62, holes_row=holes_row)
    _, _, loss, _, grads = _step(model, batch, seed=1)
    sdo = {k: v.clone().requires_grad_() for k, v in sd.items()}
    loss_ref = O.forward_loss(sdo, SMALL, batch)[0]
    loss_ref.backward()
    assert abs(loss.item() - loss_ref.item()) < 1e-2 * loss_ref.item()
    for n, g in grads.items():
        if n.endswith("attention.self.key.bias"):
            continue            # zero in exact arithmetic (a key bias shifts all scores of a query alike); both sides hold rounding noise
        want = sdo[n].grad
        assert want is not None and want.norm() > 0, n
        assert _cos(g.cpu(), want) > 0.999 and _rel_l2(g.cpu(), want) < 3e-2, (n, _cos(g.cpu(), want), _rel_l2(g.cpu(), want))


def test_lamb_training_on_the_packed_route_reduces_loss_and_is_seed_deterministic():
    """12 LAMB steps with dropout 0.1 on remove_padding(True, training=True)."""
    from deeplearningexamples_b200 import ops, training
    batch = {k: v.cuda() for k, v in _batch(4, 128, SMALL["vocab_size"], [128, 70, 33, 100], seed=71, n_labels=16).items()}
    runs = []
    for _ in range(2):
        model, opt, scaler, sched, crit, _ = training.prepare_model_and_optimizer(SMALL, torch.device("cuda"), learning_rate=2e-3,
                                                                                  warmup_proportion=0.1, max_steps=40, seed=7,
                                                                                  init_loss_scale=2 ** 10)
        model.remove_padding(True, training=True)
        ops.manual_seed(8)
        losses = []
        for _ in range(12):
            losses.append(training.take_training_step(scaler, model, crit, batch).item())
            training.take_optimizer_step(sched, opt, scaler)
        runs.append(losses)
    # the first step's loss is bitwise reproducible; later steps follow parameters updated from split-K weight gradients, whose fp32
    # atomics sum in run-dependent order
    assert runs[0][0] == runs[1][0], runs
    assert all(abs(a - b) < 1e-2 * abs(b) for a, b in zip(runs[0], runs[1])), runs
    assert runs[0][-1] < runs[0][0] - 0.3, runs[0]
