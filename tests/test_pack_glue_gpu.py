"""GPU: GLUE fine-tuning (BertForSequenceClassification).  The head kernels (dle_cls_head_fwd / dle_cls_head_bwd) against a NumPy
restatement with the hidden-dropout keep bits of test_dropout_gpu.py; the padded model against the fp32 oracle; the packed route
against the padded route on the same samples (bitwise where the arithmetic is per row); the padding-free eval route; and a captured
packed GLUE step whose replays equal eager steps."""
import types

import numpy as np
import pytest
import torch

from test_dropout_gpu import hidden_scale, reference_hidden_keep
from test_graph_replay_gpu import (_assert_same_step, _clean_state, _counter, _host_seeds, _names, _outcome, _set_counter,  # noqa: F401
                                   _state, _load, seed_log)
from test_pack_glue_cpu import sequence_classification
from test_train_packed_gpu import _assert_param_grads_agree

pytestmark = pytest.mark.gpu
bf = torch.bfloat16
DEV = torch.device("cuda", 0)
SEED = 0x8BADF00D_5EED1234
STREAM = 11
COUNTER = 5
CFG = dict(hidden_size=256, num_hidden_layers=2, num_attention_heads=4, intermediate_size=1024, vocab_size=1024,
           max_position_embeddings=512, type_vocab_size=2, hidden_act="gelu", initializer_range=0.02,
           hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
NL = 3
S, KPR = 128, 3
# k samples, a full row, a length-2 sample, an empty row, two samples
ROW_LENS = [[40, 50, 38], [128], [2, 70], [], [64, 30]]


def _cos(a, b):
    return torch.nn.functional.cosine_similarity(a.float().flatten(), b.float().flatten(), dim=0).item()


def _rel(a, b):
    return ((a.float() - b.float()).norm() / b.float().norm().clamp_min(1e-20)).item()


# ------------------------------------------------------------------------------------------------------------------------------
# head kernels against NumPy
# ------------------------------------------------------------------------------------------------------------------------------
def _seeding(mode):
    if mode == "seed_dev":
        return torch.tensor([COUNTER], dtype=torch.int64, device=DEV), COUNTER
    return None, None


def _ulp_bf16(v):
    """bf16 spacing at |v| (fp64 array)."""
    a = np.maximum(np.abs(v), 2.0 ** -126)
    return 2.0 ** (np.floor(np.log2(a)) - 7)


def _head_case(R, H, nl, dtype, p, mode, ld_pad=8, seed=0):
    from deeplearningexamples_b200 import kernels as K
    g = torch.Generator(device=DEV).manual_seed(seed + R * 7 + H + nl)
    xw = torch.randn(R, H + ld_pad, generator=g, device=DEV).to(bf)
    x = xw[:, :H]                                                            # row stride H + ld_pad
    w = (torch.randn(nl, H, generator=g, device=DEV) * 0.05).to(bf)
    b = (torch.randn(nl, generator=g, device=DEV) * 0.1).to(dtype)
    d = torch.randn(R, nl, generator=g, device=DEV).to(dtype)
    d[R // 2] = 0                                                            # a row without gradient adds exactly 0
    sdev, counter = _seeding(mode)
    kw = dict(dropout_p=p, seed=SEED, dropout_stream=STREAM, seed_dev=sdev)
    out = [K.cls_head_fwd(x, w, b, **kw), *K.cls_head_bwd(d, x, w, **kw)]
    again = [K.cls_head_fwd(x, w, b, **kw), *K.cls_head_bwd(d, x, w, **kw)]
    keep = reference_hidden_keep(R, H, SEED, STREAM, p=p, counter=counter) if p > 0 else np.ones((R, H), bool)
    return out, again, keep, (x, w, b, d)


@pytest.mark.parametrize("mode", ["host", "seed_dev"])
@pytest.mark.parametrize("p", [0.0, 0.1])
@pytest.mark.parametrize("dtype", [bf, torch.float32])
@pytest.mark.parametrize("H", [64, 768, 1024])
@pytest.mark.parametrize("nl", [1, 2, 3, 32])
def test_head_kernels_against_numpy(nl, H, dtype, p, mode):
    for R in (1, 37, 128):
        (logits, dx, dw, db), again, keep, (x, w, b, d) = _head_case(R, H, nl, dtype, p, mode)
        for a, b_ in zip((logits, dx, dw, db), again):
            assert torch.equal(a, b_), "a second launch differs"
        assert logits.dtype == dw.dtype == db.dtype == dtype and dx.dtype == bf
        sc = hidden_scale(p) if p > 0 else 1.0
        x64, w64, b64, d64 = (t.double().cpu().numpy() for t in (x, w, b, d))
        xd = np.where(keep, (x.float().cpu().numpy() * np.float32(sc)).astype(np.float64), 0.0)
        # logits: one rounding of the fp64 value, plus fp32 accumulation slack
        ref = xd @ w64.T + b64
        mag = np.abs(xd) @ np.abs(w64).T + np.abs(b64)
        got = logits.double().cpu().numpy()
        tol = (_ulp_bf16(ref) / 2 if dtype == bf else 0.0) + 1e-6 * mag + 1e-30
        assert (np.abs(got - ref) <= tol).all(), (R, np.abs(got - ref).max())
        # dx: keep * scale * d @ w; zero exactly where dropped, so backward's bits are forward's
        gd = d64 @ w64
        ref_dx = np.where(keep, gd * sc, 0.0)
        got_dx = dx.double().cpu().numpy()
        tol_dx = _ulp_bf16(ref_dx) / 2 + 1e-6 * (np.abs(d64) @ np.abs(w64)) * sc
        assert (np.abs(got_dx - ref_dx) <= tol_dx).all(), (R, np.abs(got_dx - ref_dx).max())
        assert np.array_equal(got_dx != 0, keep & (gd != 0)), "dx's zeros are not the keep bits"
        assert torch.count_nonzero(dx[R // 2]) == 0
        # dW, db: fp32 sums over rows
        ref_dw, ref_db = d64.T @ xd, d64.sum(0)
        for got_t, want in ((dw, ref_dw), (db, ref_db)):
            gt = got_t.double().cpu().numpy()
            if dtype == torch.float32:
                assert np.linalg.norm(gt - want) <= 1e-5 * np.linalg.norm(want) + 1e-30, (R, np.linalg.norm(gt - want))
            else:
                assert (np.abs(gt - want) <= _ulp_bf16(want) + 1e-6 * np.abs(want).max()).all(), (R, np.abs(gt - want).max())


@pytest.mark.parametrize("mode", ["host", "seed_dev"])
def test_head_forward_keep_bits_exact(mode):
    """Probe: W[l, c] = 1 where c % 32 == l and x[r, c] = 2^(c // 32), so logit l of row r / scale is the integer whose bit i is the
    keep bit of column 32 i + l (H = 512: 16 bits, exact in fp32)."""
    from deeplearningexamples_b200 import kernels as K
    R, H, p = 37, 512, 0.1
    c = torch.arange(H, device=DEV)
    x = (2.0 ** (c // 32)).to(bf).expand(R, H).contiguous()
    w = (c.unsqueeze(0) % 32 == torch.arange(32, device=DEV).unsqueeze(1)).to(bf)
    b = torch.zeros(32, device=DEV)
    sdev, counter = _seeding(mode)
    logits = K.cls_head_fwd(x, w, b, dropout_p=p, seed=SEED, dropout_stream=STREAM, seed_dev=sdev)
    n = torch.round(logits.double() / hidden_scale(p)).long().cpu().numpy()
    got = np.zeros((R, H), bool)
    for i in range(H // 32):
        got[:, 32 * i:32 * i + 32] = (n >> i) & 1
    want = reference_hidden_keep(R, H, SEED, STREAM, p=p, counter=counter)
    bad = np.argwhere(got != want)
    assert bad.shape[0] == 0, f"{bad.shape[0]} keep bits differ, first (row, col): {bad[:8].tolist()}"


# ------------------------------------------------------------------------------------------------------------------------------
# models
# ------------------------------------------------------------------------------------------------------------------------------
def _full_state(seed, cfg=CFG):
    from oracle import bert_oracle as O
    sd = {k: v for k, v in O.bf16_representable_params(cfg, seed=seed).items() if k.startswith("bert.")}
    g = torch.Generator().manual_seed(seed + 1)
    sd["classifier.weight"] = (torch.randn(NL, cfg["hidden_size"], generator=g) * 0.05).to(bf).float()
    sd["classifier.bias"] = (torch.randn(NL, generator=g) * 0.05).to(bf).float()
    return sd


def _model(sd, dtype=bf, cfg=CFG):
    from deeplearningexamples_b200 import glue as G
    model, _, _ = G.prepare_glue_model_and_optimizer(cfg, DEV, NL, state_dict=sd, total_steps=100, dtype=dtype)
    return model


def test_padded_model_against_fp32_oracle():
    from deeplearningexamples_b200 import glue as G
    sd = _full_state(5)
    batch = G.synthetic_glue_features(4, S, CFG["vocab_size"], NL, seed=6)
    batch["input_mask"][1] = (torch.arange(S) < S).long()                         # one full row next to ragged ones
    sdo = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    logits_ref = sequence_classification(sdo, CFG, batch["input_ids"], batch["segment_ids"], batch["input_mask"])
    loss_ref = torch.nn.CrossEntropyLoss()(logits_ref, batch["label_ids"])
    loss_ref.backward()
    model = _model(sd).train()
    b = {k: v.to(DEV) for k, v in batch.items()}
    logits = model(b["input_ids"], b["segment_ids"], b["input_mask"])
    loss = G.glue_loss(logits, b["label_ids"])
    loss.backward()
    lg = logits.float().cpu()
    assert _rel(lg, logits_ref) < 1e-2 and (lg - logits_ref).abs().max() / logits_ref.abs().max() < 2e-2, (lg, logits_ref)
    assert abs(loss.item() - loss_ref.item()) < 5e-3 * loss_ref.item(), (loss.item(), loss_ref.item())
    for n, p in model.named_parameters():
        want = sdo[n].grad
        if want is None or n.endswith("key.bias") or want.norm() == 0:
            continue
        got = p.grad.float().cpu()
        assert _cos(got, want) > 0.999 and _rel(got, want) < 3e-2, (n, _cos(got, want), _rel(got, want))


def _samples(lens, seed):
    from deeplearningexamples_b200 import glue as G, packing
    src = G.synthetic_glue_features(len(lens), S, CFG["vocab_size"], NL, seed=seed, min_len=5, max_len=S)
    out = []
    for i, n in enumerate(lens):
        ids = src["input_ids"][i, :n].clone()
        ids[-1] = 102
        out.append(packing.GlueSample(ids.numpy(), src["segment_ids"][i, :n].numpy(), int(src["label_ids"][i]), i))
    return out


def _packed(row_lens, seed, B=None):
    """A packed GLUE batch whose row r holds samples of lengths row_lens[r], and the samples in order."""
    from deeplearningexamples_b200 import packing
    samples = _samples([n for r in row_lens for n in r], seed)
    rows, i = [], 0
    for r in row_lens:
        rows.append(list(range(i, i + len(r))))
        i += len(r)
    return packing.to_glue_batch(samples, rows, B or len(row_lens), S, KPR), samples


def _padded_by_slot(packed, samples):
    """The padded batch with one row per slot of `packed` (so the pooler and head see the same number of rows): a slot's sample
    right-padded, and for an empty slot a two-token filler row with label -100."""
    R = packed["label_ids"].shape[0]
    b = {"input_ids": torch.zeros(R, S, dtype=torch.long), "segment_ids": torch.zeros(R, S, dtype=torch.long),
         "input_mask": torch.zeros(R, S, dtype=torch.long), "label_ids": torch.full((R,), -100, dtype=torch.long)}
    for slot, e in enumerate(packed.example_index):
        if e < 0:
            b["input_ids"][slot, :2] = torch.tensor([101, 102])
            b["input_mask"][slot, :2] = 1
            continue
        s = samples[int(e)]
        n = len(s)
        b["input_ids"][slot, :n] = torch.from_numpy(s.input_ids)
        b["segment_ids"][slot, :n] = torch.from_numpy(s.segment_ids)
        b["input_mask"][slot, :n] = 1
        b["label_ids"][slot] = s.label
    return b


def _slots(packed):
    """(slot, flat positions in the packed batch) of each sample."""
    am = packed["input_mask"]
    out = []
    for r in range(am.shape[0]):
        for j in range(1, KPR + 1):
            where = torch.nonzero(am[r] == j).squeeze(-1)
            if where.numel():
                out.append((r * KPR + j - 1, r * S + where))
    return out


KEYS = ("input_ids", "segment_ids", "input_mask")


@pytest.mark.parametrize("dtype", [bf, torch.float32])
def test_packed_eval_logits_equal_padded_logits(dtype):
    model = _model(_full_state(31), dtype).eval()
    packed, samples = _packed(ROW_LENS, seed=32)
    padded = _padded_by_slot(packed, samples)
    with torch.no_grad():
        l_pad = model(*(padded[k].to(DEV) for k in KEYS))
        model.pack_sequences(KPR)
        l_pk = model(*(packed[k].to(DEV) for k in KEYS))
        model.pack_sequences(0)
    assert l_pk.shape == (len(ROW_LENS) * KPR, NL) and l_pk.dtype == l_pad.dtype == dtype
    used = packed.example_index >= 0
    assert torch.equal(l_pk[torch.as_tensor(used, device=DEV)], l_pad[torch.as_tensor(used, device=DEV)])
    assert bool(l_pk.isfinite().all())


def _glue_step(model, batch):
    """Forward + backward in train mode: (per-slot CE terms, mean loss, gradient at the embedding output, parameter gradients)."""
    from deeplearningexamples_b200 import glue as G, ops
    emb = []

    def hook(mod, inp, out):
        out.retain_grad()
        emb.append(out)
    h = model.bert.embeddings.register_forward_hook(hook)
    try:
        ops.manual_seed(5)
        b = {k: v.to(DEV) for k, v in batch.items()}
        logits = model(b["input_ids"], b["segment_ids"], b["input_mask"])
        rows = torch.nn.CrossEntropyLoss(reduction="none")(logits.float(), b["label_ids"])
        loss = G.glue_loss(logits, b["label_ids"])
        loss.backward()
    finally:
        h.remove()
    grads = {n: p.grad.detach().clone() for n, p in model.named_parameters() if p.grad is not None}
    model.zero_grad(set_to_none=True)
    return rows.detach(), loss.detach(), emb[0].grad.detach().reshape(-1, CFG["hidden_size"]).clone(), grads


def test_packed_training_step_equals_padded_step():
    model = _model(_full_state(41)).train()
    packed, samples = _packed(ROW_LENS, seed=42)
    padded = _padded_by_slot(packed, samples)
    rows_pad, l_pad, e_pad, g_pad = _glue_step(model, padded)
    model.pack_sequences(KPR)
    rows_pk, l_pk, e_pk, g_pk = _glue_step(model, packed)
    model.pack_sequences(0)
    sample_tokens = torch.zeros(e_pk.shape[0], dtype=torch.bool, device=DEV)
    for slot, fp in _slots(packed):
        n = fp.numel()
        assert torch.equal(rows_pk[slot], rows_pad[slot]), slot
        assert torch.equal(e_pk[fp.to(DEV)], e_pad[slot * S:slot * S + n]), slot
        sample_tokens[fp.to(DEV)] = True
    assert torch.count_nonzero(e_pk[~sample_tokens]) == 0                     # the tail's gradient is exactly zero
    assert abs(l_pk.item() - l_pad.item()) <= 1e-5 * abs(l_pad.item())
    _assert_param_grads_agree({n: g for n, g in g_pk.items() if not n.endswith("key.bias")},
                              {n: g for n, g in g_pad.items() if not n.endswith("key.bias")}, 0.9999, 1e-2)


def test_padding_free_eval_logits_equal_padded_logits():
    from deeplearningexamples_b200 import glue as G
    model = _model(_full_state(71)).eval()
    b = {k: v.to(DEV) for k, v in G.synthetic_glue_features(6, S, CFG["vocab_size"], NL, seed=72).items()}
    with torch.no_grad():
        want = model(*(b[k] for k in KEYS))
        model.remove_padding(True)
        got = model(*(b[k] for k in KEYS))
        model.remove_padding(False)
    assert bool((b["input_mask"] == 0).any()) and torch.equal(got, want)


# ------------------------------------------------------------------------------------------------------------------------------
# CUDA graph
# ------------------------------------------------------------------------------------------------------------------------------
DROP = dict(CFG, hidden_dropout_prob=0.1, attention_probs_dropout_prob=0.1)
GRAPH_ROWS = [[[60, 60], [128], [40, 40, 40], [100]],
              [[30, 30, 30], [], [128], [1, 120]],
              [[128], [64, 64], [20, 30, 70], []],
              [[], [90, 20, 1], [30], [100, 28]]]


def _glue_arm(sd):
    """The GLUE training state in the shape test_graph_replay_gpu.py's helpers read (FusedAdam without a loss scaler)."""
    from deeplearningexamples_b200 import glue as G, ops
    ops.manual_seed(42)                             # same dropout stream ids in both arms
    model, opt, sched = G.prepare_glue_model_and_optimizer(DROP, DEV, NL, state_dict=sd, total_steps=50, learning_rate=1e-4)
    model.train()
    model.pack_sequences(KPR)
    scaler = types.SimpleNamespace(_scale=torch.ones(1, device=DEV), _growth_tracker=torch.zeros(1, dtype=torch.int32, device=DEV))
    return types.SimpleNamespace(model=model, opt=opt, sched=sched, scaler=scaler, skipped_acc=None,
                                 loss_acc=torch.zeros(1, dtype=torch.float32, device=DEV))


def _step(arm, batch):
    from deeplearningexamples_b200 import glue as G
    G.glue_training_step(arm.model, arm.opt, arm.sched, batch, arm.loss_acc)


def test_replayed_packed_glue_step_matches_eager(seed_log):
    """The whole packed GLUE step (FusedAdam, device-side schedule, dropout 0.1 in the encoder and the head) captured once; before
    each of three replays a differently packed batch is copied into the static buffers.  Each replay equals eager steps from the same
    state, which draw the host seeds the capture froze."""
    from deeplearningexamples_b200 import ops, training as T
    sd = _full_state(61)
    batches = [{k: v.to(DEV) for k, v in _packed(r, seed=62 + i)[0].items()} for i, r in enumerate(GRAPH_ROWS)]
    g = _glue_arm(sd)
    g.static = {k: v.clone() for k, v in batches[0].items()}
    starts = []

    def one_step():
        starts.append(len(seed_log))
        _step(g, g.static)
    g.graph = T.capture_step_graph(one_step, warmup_iters=3)
    seeds = list(seed_log[starts[-1]:])
    assert len(seeds) == 1 + 3 * DROP["num_hidden_layers"] + 1                # embeddings, 3 per layer, the head
    e = _glue_arm(sd)
    for _ in range(3):
        _step(e, batches[0])
    names = _names(g)
    replay_losses = []
    for i, batch in enumerate(batches[1:]):
        pre, c0 = _state(g), _counter()
        runs = []
        for _ in range(2):
            _load(e, pre)
            _set_counter(c0)
            e.loss_acc.zero_()
            with _host_seeds(seeds):
                _step(e, batch)
            runs.append(_outcome(e, pre, [e.loss_acc.clone()]))
        for k in g.static:
            g.static[k].copy_(batch[k])
        _set_counter(c0)
        g.loss_acc.zero_()
        g.graph.replay()
        assert _counter() == c0 + 1
        got = _outcome(g, pre, [g.loss_acc.clone()])
        _assert_same_step(got, runs[0], runs[1], names, f"replay {i}")
        assert got["found_inf"].item() == 0.0 and got["loss"].isfinite().all()
        replay_losses.append(got["loss"].item())
        # the head's mask is part of the step: a wrong head seed changes the loss
        wrong = seeds[:-1] + [seeds[-1] ^ 0x5A5A]
        _load(e, pre)
        _set_counter(c0)
        e.loss_acc.zero_()
        with _host_seeds(wrong):
            _step(e, batch)
        assert not torch.equal(e.loss_acc, got["loss"].reshape(1))
    assert len(set(replay_losses)) == 3, replay_losses
    ops.check_device_errors()
    del g, e
