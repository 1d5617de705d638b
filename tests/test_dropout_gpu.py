"""Dropout-on training checked exactly and against fp32.

1. Keep bits.  Every hidden-dropout kernel (the GEMM epilogue EPI_BIAS_DROPOUT_RESIDUAL, add_ln_fwd and add_ln_bwd in their one-warp
   and two-warp families, embed_ln_fwd) is pinned bit for bit to a NumPy restatement of common.cuh (dropout_keep32 / dropout_keep8,
   dropout_thresh16, effective_seed).  The layer's forward draws its hidden masks in the GEMM epilogue and its backward draws them
   again in add_ln_bwd, so the two are also compared with each other directly.
2. Gradients.  BertLayer (fused, modular and packed) and the embeddings run with dropout 0.1 and a non-zero step counter, against the
   fp32 oracle given the restated keep masks.  In each test the same oracle with one site's mask drawn from the wrong stream must miss
   the kernel by far, which shows the comparison can see a wrong mask.
3. Graph replay.  A captured whole training step draws each replay's embedding mask from the device step counter, with the host seed
   frozen at capture.

Keep bits are compared exactly: no tolerance is applied to a mask.  fp32 comparisons use the bars of the other oracle tests: relative
L2 < 1e-2 on forward outputs; cosine similarity > 0.999 and relative L2 < 3e-2 on gradients."""
import numpy as np
import pytest
import torch

from test_attention_wgmma_gpu import _philox4x32_7, _thresh15, reference_keep

pytestmark = pytest.mark.gpu
bf = torch.bfloat16
M32 = 0xFFFFFFFF
MASK64 = (1 << 64) - 1
GOLDEN = 0x9E3779B97F4A7C15            # effective_seed's multiplier of the device step counter
P = 0.1
SEED = 0x8BADF00D_5EED1234             # both 32-bit halves non-zero
STREAM = 9
COUNTER = 7
LN_T = 5000                            # ragged, and above one grid sweep of either LayerNorm family (132 SMs x 16 rows)


# ------------------------------------------------------------------------------------------------------------------------------
# NumPy restatement of the hidden-dropout key (common.cuh)
# ------------------------------------------------------------------------------------------------------------------------------
def thresh16(p):
    """dropout_thresh16 in float32 arithmetic."""
    t = np.float32(p) * np.float32(65536.0) + np.float32(0.5)
    return 0 if t <= 0 else (65535 if t >= 65535 else int(t))


def hidden_scale(p):
    return float(np.float32(1.0) / (np.float32(1.0) - np.float32(p)))


def attn_scale(p):
    """attn_drop_params: p quantised to 1/32768."""
    return float(np.float32(1.0) / (np.float32(1.0) - np.float32(_thresh15(p)) / np.float32(32768.0)))


def effective_seed(seed, counter):
    return seed if counter is None else (seed + counter * GOLDEN) & MASK64


def keep32(seed, stream, groups, t16):
    """dropout_keep32(seed, stream, g, t16) of every group g (uint64 array holding 32-bit words): one Philox4x32-7 block per group;
    word r_w seeds an LCG whose states s_0 = r_w, s_1, ... give bits 8w + k = (s_k >= t16 << 16)."""
    r = _philox4x32_7(groups & np.uint64(M32), groups >> np.uint64(32), np.full_like(groups, stream), np.full_like(groups, 0x5EED32),
                      seed & M32, (seed >> 32) & M32)
    t = np.uint64(t16 << 16)
    m = np.zeros_like(groups)
    for w in range(4):
        s = r[w]
        for k in range(8):
            m |= (s >= t).astype(np.uint64) << np.uint64(8 * w + k)
            s = (s * np.uint64(747796405) + np.uint64(2891336453)) & np.uint64(M32)
    return m


def reference_hidden_keep(rows, width, seed, stream, p=P, counter=None):
    """bool [rows, width]: flat element e = row * width + col is kept iff bit e & 31 of keep32(seed_eff, stream, e >> 5) is set."""
    n = rows * width
    assert n % 32 == 0
    m = keep32(effective_seed(seed, counter), stream, np.arange(n // 32, dtype=np.uint64), thresh16(p))
    return np.unpackbits(m.astype("<u4").view(np.uint8), bitorder="little").astype(bool).reshape(rows, width)


def test_restatement_threshold_and_seed_arithmetic():
    assert thresh16(0.1) == 6554 and _thresh15(0.1) == 3277
    assert effective_seed(SEED, None) == SEED
    assert effective_seed(MASK64, 1) == GOLDEN - 1                      # wraps mod 2^64
    m = reference_hidden_keep(1, 64, 1, 2, p=0.0)                        # t16 = 0 keeps everything
    assert m.all()


# ------------------------------------------------------------------------------------------------------------------------------
# exact keep bits of every hidden-dropout kernel
# ------------------------------------------------------------------------------------------------------------------------------
def _k():
    from deeplearningexamples_b200 import kernels
    return kernels


def _seeding(mode):
    """(seed_dev tensor or None, counter the kernels mix in or None)."""
    if mode == "seed_dev":
        return torch.tensor([COUNTER], dtype=torch.int64, device="cuda"), COUNTER
    return None, None


def _kept_value(p=P):
    return torch.tensor(hidden_scale(p)).to(bf).item()


def _assert_two_valued(t, what):
    """t holds only 0 and the scaled 1; returns the keep mask as a NumPy bool array."""
    kv = _kept_value()
    bad = ~((t == 0) | (t == kv))
    assert not bool(bad.any()), f"{what}: {int(bad.sum())} values are neither 0 nor {kv}, e.g. {t[bad][:4].tolist()}"
    return (t != 0).cpu().numpy()


def _assert_same_bits(got, want, what, valid=None):
    diff = got != want
    if valid is not None:
        diff &= valid
    bad = np.argwhere(diff)
    assert bad.shape[0] == 0, f"{what}: {bad.shape[0]} keep bits differ, first (row, col): {bad[:8].tolist()}"


def _gemm_keep(M, N, seed, stream, seed_dev, tile_n=0):
    """Keep mask of the GEMM epilogue: A = 0, bias = 1, aux = 0, so each output is 0 or bf16(1 / (1 - p))."""
    from deeplearningexamples_b200 import _lib as L
    k = _k()
    g = torch.Generator(device="cuda").manual_seed(M + N)
    a = torch.zeros(M, 64, device="cuda", dtype=bf)
    b = torch.randn(N, 64, generator=g, device="cuda").to(bf)
    out = k.gemm(a, b, epilogue=L.EPI_BIAS_DROPOUT_RESIDUAL, bias=torch.ones(N, device="cuda", dtype=bf),
                 aux=torch.zeros(M, N, device="cuda", dtype=bf), dropout_p=P, seed=seed, seed_dev=seed_dev, dropout_stream=stream,
                 tile_n=tile_n)
    return _assert_two_valued(out, f"gemm M={M} N={N} tile_n={tile_n}")


def _ln_bwd_keep(T, H, seed, stream, seed_dev):
    """Keep mask of add_ln_bwd: dx = dz * scale where kept, else 0.  Returns (keep, valid = dz != 0)."""
    k = _k()
    g = torch.Generator(device="cuda").manual_seed(T + H)
    z = torch.randn(T, H, generator=g, device="cuda").to(bf)
    gamma = (1.0 + 0.1 * torch.randn(H, generator=g, device="cuda")).to(bf)
    beta = torch.zeros(H, device="cuda", dtype=bf)
    _, _, mean, rstd = k.add_ln_fwd(z, gamma, beta)
    dy = torch.randn(T, H, generator=g, device="cuda").to(bf)
    dz, dx, _, _, _ = k.add_ln_bwd(dy, z, mean, rstd, gamma, dropout_p=P, seed=seed, dropout_stream=stream, seed_dev=seed_dev)
    valid = (dz != 0).cpu().numpy()
    assert valid.mean() > 0.99, valid.mean()
    return (dx != 0).cpu().numpy(), valid


GEMM_SHAPES = [(tile_n, N, M) for tile_n in (128, 0) for N in (256, 768, 1024) for M in (130, 1000)]


@pytest.mark.parametrize("seeding", ["seed_dev", "host"])
@pytest.mark.parametrize("tile_n,N,M", GEMM_SHAPES + [(128, 1024, 16384), (0, 1024, 16384)])
def test_gemm_epilogue_keep_bits(tile_n, N, M, seeding):
    seed_dev, counter = _seeding(seeding)
    got = _gemm_keep(M, N, SEED, STREAM, seed_dev, tile_n)
    want = reference_hidden_keep(M, N, SEED, STREAM, counter=counter)
    _assert_same_bits(got, want, f"gemm tile_n={tile_n}")
    if M * N >= 4 << 20:
        assert abs(got.mean() - (1.0 - thresh16(P) / 65536.0)) < 1e-3, got.mean()


@pytest.mark.parametrize("seeding", ["seed_dev", "host"])
@pytest.mark.parametrize("H", [256, 768, 512, 1024])                   # one-warp kernels, then two-warp kernels
def test_add_ln_fwd_keep_bits(H, seeding):
    k = _k()
    seed_dev, counter = _seeding(seeding)
    x = torch.ones(LN_T, H, device="cuda", dtype=bf)
    gamma, beta = torch.ones(H, device="cuda", dtype=bf), torch.zeros(H, device="cuda", dtype=bf)
    _, z, _, _ = k.add_ln_fwd(x, gamma, beta, residual=torch.zeros_like(x), dropout_p=P, seed=SEED, dropout_stream=STREAM,
                              seed_dev=seed_dev)
    got = _assert_two_valued(z, f"add_ln_fwd H={H}")
    _assert_same_bits(got, reference_hidden_keep(LN_T, H, SEED, STREAM, counter=counter), f"add_ln_fwd H={H}")


@pytest.mark.parametrize("seeding", ["seed_dev", "host"])
@pytest.mark.parametrize("H", [256, 768, 512, 1024])
def test_add_ln_bwd_keep_bits(H, seeding):
    seed_dev, counter = _seeding(seeding)
    got, valid = _ln_bwd_keep(LN_T, H, SEED, STREAM, seed_dev)
    _assert_same_bits(got, reference_hidden_keep(LN_T, H, SEED, STREAM, counter=counter), f"add_ln_bwd H={H}", valid)


@pytest.mark.parametrize("seeding", ["seed_dev", "host"])
@pytest.mark.parametrize("H", [256, 512, 768, 1024])
def test_embed_ln_fwd_keep_bits(H, seeding):
    k = _k()
    seed_dev, counter = _seeding(seeding)
    B, S, V, NP, NT = 10, 500, 64, 512, 2
    g = torch.Generator(device="cuda").manual_seed(H)
    ids = torch.randint(0, V, (B, S), generator=g, device="cuda")
    tts = torch.randint(0, NT, (B, S), generator=g, device="cuda")
    word, pos, typ = (torch.randn(n, H, generator=g, device="cuda").to(bf) for n in (V, NP, NT))
    gamma, beta = torch.zeros(H, device="cuda", dtype=bf), torch.ones(H, device="cuda", dtype=bf)   # y = 1 before dropout
    y, _, _, _ = k.embed_ln_fwd(ids, tts, word, pos, typ, gamma, beta, dropout_p=P, seed=SEED, dropout_stream=STREAM,
                                seed_dev=seed_dev)
    got = _assert_two_valued(y, f"embed_ln_fwd H={H}")
    _assert_same_bits(got, reference_hidden_keep(B * S, H, SEED, STREAM, counter=counter), f"embed_ln_fwd H={H}")


@pytest.mark.parametrize("H", [256, 768, 512, 1024])
def test_gemm_forward_mask_equals_add_ln_bwd_mask(H):
    """The encoder layer's hand-off: forward drops in the GEMM epilogue (dropout_keep32 over N = H), backward regenerates the mask in
    add_ln_bwd (dropout_keep8); with the same seed, stream and counter the two must agree on every element."""
    seed_dev, _ = _seeding("seed_dev")
    T = 3000
    fwd = _gemm_keep(T, H, SEED, STREAM, seed_dev)
    bwd, valid = _ln_bwd_keep(T, H, SEED, STREAM, seed_dev)
    _assert_same_bits(bwd, fwd, f"H={H}: add_ln_bwd against the GEMM epilogue", valid)


# ------------------------------------------------------------------------------------------------------------------------------
# dropout-on gradients against fp32 with the known masks
# ------------------------------------------------------------------------------------------------------------------------------
SMALL = dict(hidden_size=256, num_hidden_layers=2, num_attention_heads=4, intermediate_size=1024, vocab_size=1024,
             max_position_embeddings=512, type_vocab_size=2, hidden_act="gelu", initializer_range=0.02,
             hidden_dropout_prob=P, attention_probs_dropout_prob=P)


def _rel_l2(got, want):
    return ((got.float() - want.float()).norm() / want.float().norm().clamp_min(1e-12)).item()


def _cos(got, want):
    return torch.nn.functional.cosine_similarity(got.float().flatten(), want.float().flatten(), dim=0).item()


def _assert_grad_close(got, want, name):
    got = got.float().cpu()
    assert _cos(got, want) > 0.999 and _rel_l2(got, want) < 3e-2, (name, _cos(got, want), _rel_l2(got, want))


@pytest.fixture
def seed_log(monkeypatch):
    """The host seeds the dropout call sites draw, in order (ops.next_seed, logged)."""
    from deeplearningexamples_b200 import ops
    drawn, real = [], ops.next_seed

    def logged():
        s = real()
        drawn.append(s)
        return s
    monkeypatch.setattr(ops, "next_seed", logged)
    return drawn


@pytest.fixture
def step_counter():
    """The device step counter set to COUNTER for the test, and back to 0 after it."""
    from deeplearningexamples_b200 import ops
    ops.manual_seed(1234)
    c = ops.step_counter(torch.device("cuda"))
    c.fill_(COUNTER)
    yield c
    c.zero_()


def _layer(seed):
    """A SMALL BertLayer in bf16, train mode, with random non-trivial weights, biases and LayerNorm affines."""
    from deeplearningexamples_b200 import modeling
    layer = modeling.BertLayer(modeling.BertConfig.from_dict(SMALL)).cuda().to(bf).train()
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for n, p in layer.named_parameters():
            v = torch.randn(p.shape, generator=g) * 0.05
            p.copy_((v + 1.0) if n.endswith("LayerNorm.weight") else v)
    return layer


def _layer_sites(layer, seeds):
    """[(effective seed, stream)] of the attention, attention-output and output dropout sites, in the order they draw seeds."""
    att, so, out = layer.attention.self, layer.attention.output, layer.output
    assert len(seeds) == 3, seeds
    return [(effective_seed(s, COUNTER), sid) for s, sid in zip(seeds, (att._stream_id, so._stream_id, out._stream_id))]


def _oracle_params(layer):
    return {n: p.detach().float().cpu().requires_grad_() for n, p in layer.named_parameters()}


def _assert_layer_grads(layer, sd, dx, dx_ref):
    _assert_grad_close(dx, dx_ref, "dx")
    for n, p in layer.named_parameters():
        if n.endswith("attention.self.key.bias"):
            continue            # zero in exact arithmetic (a key bias shifts all scores of a query alike); both sides hold rounding noise
        assert sd[n].grad is not None and sd[n].grad.norm() > 0, n
        _assert_grad_close(p.grad, sd[n].grad, n)


@pytest.mark.parametrize("modular", [False, True], ids=["fused", "modular"])
def test_layer_padded_dropout_vs_fp32(modular, seed_log, step_counter):
    """ops.BertLayerFn (fused) or the module-by-module path (DenseDropoutAddLNFn) with p_attn = p_hid = 0.1 on a ragged batch.  The
    hidden masks are keyed by memory row: the encoder's [S, B, H] view of a batch-first buffer puts token (b, s) at row b*S + s."""
    from oracle import bert_oracle as O
    layer = _layer(31)
    layer.force_modular = modular
    B, S, H, A = 4, 128, SMALL["hidden_size"], SMALL["num_attention_heads"]
    keep = torch.arange(S).unsqueeze(0) < torch.tensor([128, 77, 1, 100]).unsqueeze(1)
    mask = ((~keep).float() * -10000.0).view(B, 1, 1, S)
    g = torch.Generator().manual_seed(32)
    x0 = torch.randn(B, S, H, generator=g).to(bf)
    dy = torch.randn(B, S, H, generator=g).to(bf)

    x = x0.cuda().requires_grad_()
    y = layer(x.transpose(0, 1), mask.cuda()).transpose(0, 1)
    y.backward(dy.cuda())
    (seed_a, sid_a), (seed_1, sid_1), (seed_2, sid_2) = _layer_sites(layer, seed_log)

    def reference(sd, xr, wrong_site=None):
        ak = torch.from_numpy(reference_keep(B, S, A, P, seed_a, sid_a + (wrong_site == 0)))
        hk = [torch.from_numpy(reference_hidden_keep(B * S, H, s, sid + (wrong_site == i))).view(B, S, H).transpose(0, 1)
              for i, (s, sid) in ((1, (seed_1, sid_1)), (2, (seed_2, sid_2)))]
        return O.bert_layer(sd, "", xr.transpose(0, 1), mask, A, ak, attn_scale(P), hk, hidden_scale(P)).transpose(0, 1)

    sd = _oracle_params(layer)
    xr = x0.float().requires_grad_()
    y_ref = reference(sd, xr)
    y_ref.backward(dy.float())
    assert _rel_l2(y.cpu(), y_ref.detach()) < 1e-2, _rel_l2(y.cpu(), y_ref.detach())
    _assert_layer_grads(layer, sd, x.grad, xr.grad)
    with torch.no_grad():                        # control: the output dropout's mask drawn from the neighbouring stream
        y_bad = reference(sd, xr, wrong_site=2)
    assert _rel_l2(y.cpu(), y_bad) > 0.1, _rel_l2(y.cpu(), y_bad)


def test_layer_packed_dropout_vs_fp32(seed_log, step_counter):
    """ops.BertLayerPackedFn (BertLayer.forward_packed) with p_attn = p_hid = 0.1 on packed sequences from a batch with a row with
    holes and a length-1 row.  Hidden masks are keyed by packed row; attention masks by (sequence, head, in-sequence query,
    in-sequence key) with drop_stride = S rounded up to 64.  The fp32 reference attends within each packed sequence."""
    from oracle import bert_oracle as O
    layer = _layer(41)
    B, S, H, A = 4, 200, SMALL["hidden_size"], SMALL["num_attention_heads"]
    stride = (S + 63) // 64 * 64
    g = torch.Generator().manual_seed(42)
    keep = torch.arange(S).unsqueeze(0) < torch.tensor([200, S, 1, 150]).unsqueeze(1)
    keep[1] = torch.rand(S, generator=g) < 0.6                              # a row with holes
    keep[1, 0] = True
    lens = keep.sum(1)
    cu = [0] + torch.cumsum(lens, 0).tolist()
    T = cu[-1]
    x0 = torch.randn(T, H, generator=g).to(bf)
    dy = torch.randn(T, H, generator=g).to(bf)

    x = x0.cuda().requires_grad_()
    y = layer.forward_packed(x, torch.tensor(cu, dtype=torch.int32, device="cuda"), int(lens.max()), stride)
    y.backward(dy.cuda())
    (seed_a, sid_a), (seed_1, sid_1), (seed_2, sid_2) = _layer_sites(layer, seed_log)

    def reference(sd, xr, wrong_site=None):
        ak = torch.from_numpy(reference_keep(B, stride, A, P, seed_a, sid_a + (wrong_site == 0)))
        h1 = torch.from_numpy(reference_hidden_keep(T, H, seed_1, sid_1 + (wrong_site == 1)))
        h2 = torch.from_numpy(reference_hidden_keep(T, H, seed_2, sid_2 + (wrong_site == 2)))
        outs = []
        for b in range(B):
            r0, n = cu[b], cu[b + 1] - cu[b]
            rows = slice(r0, r0 + n)
            outs.append(O.bert_layer(sd, "", xr[rows].unsqueeze(1), torch.zeros(1, 1, 1, n), A, ak[b:b + 1, :, :n, :n], attn_scale(P),
                                     (h1[rows].unsqueeze(1), h2[rows].unsqueeze(1)), hidden_scale(P)).squeeze(1))
        return torch.cat(outs)

    sd = _oracle_params(layer)
    xr = x0.float().requires_grad_()
    y_ref = reference(sd, xr)
    y_ref.backward(dy.float())
    assert _rel_l2(y.cpu(), y_ref.detach()) < 1e-2, _rel_l2(y.cpu(), y_ref.detach())
    _assert_layer_grads(layer, sd, x.grad, xr.grad)
    with torch.no_grad():                        # control: the output dropout's mask drawn from the neighbouring stream
        y_bad = reference(sd, xr, wrong_site=2)
    assert _rel_l2(y.cpu(), y_bad) > 0.1, _rel_l2(y.cpu(), y_bad)


def test_embedding_dropout_vs_fp32(seed_log, step_counter):
    """ops.EmbeddingLNFn with p = 0.1: y and the gradients of the three tables and the LayerNorm affine, whose backward
    (embed_ln_bwd_kernel) regenerates the forward's mask."""
    from deeplearningexamples_b200 import ops
    from oracle import bert_oracle as O
    B, S, H, V, NP, NT, stream = 4, 128, 256, 64, 512, 2, 13
    g = torch.Generator().manual_seed(51)
    ids = torch.randint(0, V, (B, S), generator=g)                        # V < B*S: rows of dword sum many tokens
    tts = torch.randint(0, NT, (B, S), generator=g)
    params = {"word_embeddings.weight": torch.randn(V, H, generator=g) * 0.5,
              "position_embeddings.weight": torch.randn(NP, H, generator=g) * 0.5,
              "token_type_embeddings.weight": torch.randn(NT, H, generator=g) * 0.5,
              "LayerNorm.weight": 1.0 + 0.1 * torch.randn(H, generator=g),
              "LayerNorm.bias": 0.1 * torch.randn(H, generator=g)}
    params = {n: v.to(bf).float() for n, v in params.items()}             # fp32 parameters holding bf16 values
    dy = torch.randn(B * S, H, generator=g).to(bf)

    dev = {n: v.cuda().requires_grad_() for n, v in params.items()}
    y = ops.EmbeddingLNFn.apply(ids.cuda(), tts.cuda(), dev["word_embeddings.weight"], dev["position_embeddings.weight"],
                                dev["token_type_embeddings.weight"], dev["LayerNorm.weight"], dev["LayerNorm.bias"], P, 1e-12, stream)
    y.backward(dy.cuda())
    assert len(seed_log) == 1
    seed = effective_seed(seed_log[0], COUNTER)

    def reference(sd, wrong_stream=False):
        keep = torch.from_numpy(reference_hidden_keep(B * S, H, seed, stream + wrong_stream)).view(B, S, H)
        return O.embeddings(sd, ids, tts, prefix="", drop_keep=keep, drop_scale=hidden_scale(P)).view(B * S, H)

    sd = {n: v.clone().requires_grad_() for n, v in params.items()}
    y_ref = reference(sd)
    y_ref.backward(dy.float())
    assert _rel_l2(y.cpu(), y_ref.detach()) < 1e-2, _rel_l2(y.cpu(), y_ref.detach())
    for n in params:
        _assert_grad_close(dev[n].grad, sd[n].grad, n)
    with torch.no_grad():                        # control: the mask drawn from the neighbouring stream
        y_bad = reference(sd, wrong_stream=True)
    assert _rel_l2(y.cpu(), y_bad) > 0.1, _rel_l2(y.cpu(), y_bad)


# ------------------------------------------------------------------------------------------------------------------------------
# the step counter under graph replay
# ------------------------------------------------------------------------------------------------------------------------------
def test_graph_replay_draws_embedding_masks_from_the_step_counter(seed_log):
    """One forward + backward step of a SMALL BertForPreTraining with dropout 0.1, captured as a CUDA graph and replayed twice: the
    host seed is frozen at capture, and each replay's embedding mask is the one of that seed at the counter value the replay
    advanced to."""
    from deeplearningexamples_b200 import modeling, ops, training
    from oracle import bert_oracle as O
    ops.manual_seed(61)
    model = modeling.BertForPreTraining(modeling.BertConfig.from_dict(SMALL)).cuda().to(bf)
    crit = training.BertPretrainingCriterion(SMALL["vocab_size"])
    B, S, H = 2, 128, SMALL["hidden_size"]
    batch = {k: v.cuda() for k, v in O.synthetic_batch(B, S, SMALL["vocab_size"], 10, seed=62, full_mask=False).items()}
    model.eval()
    with torch.no_grad():
        nonzero = (model.bert.embeddings(batch["input_ids"], batch["token_type_ids"]) != 0).cpu().numpy().reshape(B * S, H)
    assert nonzero.mean() > 0.99
    model.train()
    outs, starts = [], []
    # detached: the list keeps each output's memory alive (the captured one is the graph's static tensor) but not its autograd graph
    hook = model.bert.embeddings.register_forward_hook(lambda mod, inp, out: outs.append(out.detach()))

    def step():
        starts.append(len(seed_log))
        model.zero_grad(set_to_none=True)
        scores, nsp = model(batch["input_ids"], batch["token_type_ids"], batch["attention_mask"], batch["labels"])
        crit(scores, nsp, batch["labels"], batch["next_sentence_labels"]).backward()
    try:
        graph = training.capture_step_graph(step, warmup_iters=2)
    finally:
        hook.remove()
    host_seed, static = seed_log[starts[-1]], outs[-1]                   # the embedding draws first; its output in the graph's memory
    assert len(seed_log) - starts[-1] == 1 + 3 * SMALL["num_hidden_layers"]
    stream = model.bert.embeddings._stream_id
    counter = ops.step_counter(torch.device("cuda"))
    masks, last = [], int(counter.item())
    for _ in range(2):
        graph.replay()
        torch.cuda.synchronize()
        c = int(counter.item())
        assert c == last + 1, (c, last)
        got = (static != 0).cpu().numpy().reshape(B * S, H)
        want = reference_hidden_keep(B * S, H, host_seed, stream, counter=c)
        _assert_same_bits(got, want, f"embedding mask of the replay at counter {c}", nonzero)
        masks.append(got)
        last = c
    assert (masks[0] != masks[1])[nonzero].mean() > 0.1
    counter.zero_()
