"""GPU: SWAG fine-tuning (BertForMultipleChoice).  The padded model against the fp32 oracle; the packed route against the padded route
on the same examples (bitwise where the arithmetic is per row), in bf16 and fp32 parameters, at a small width and at BERT-large widths;
the padding-free eval route; a captured packed SWAG step whose replays equal eager steps, schedule included; and the refusals."""
import types

import pytest
import torch

from test_graph_replay_gpu import (_assert_same_step, _clean_state, _counter, _host_seeds, _names, _outcome, _set_counter,  # noqa: F401
                                   _state, _load, seed_log)
from test_pack_swag_cpu import multiple_choice
from test_train_packed_gpu import _assert_param_grads_agree

pytestmark = pytest.mark.gpu
bf = torch.bfloat16
DEV = torch.device("cuda", 0)
CFG = dict(hidden_size=256, num_hidden_layers=2, num_attention_heads=4, intermediate_size=1024, vocab_size=1024,
           max_position_embeddings=512, type_vocab_size=2, hidden_act="gelu", initializer_range=0.02,
           hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
WIDE = dict(CFG, hidden_size=1024, num_attention_heads=16, intermediate_size=4096)      # two layers at BERT-large widths
C = 4
S, KPR = 256, 8                     # packed rows of 256 tokens, two examples of four choices each; padded choice rows of 256 tokens
# per row, the examples' choice lengths: k/C examples, an example that fills S exactly, an empty row, a real group then an empty one
ROW_LENS = [[[20, 30, 25, 40], [31, 19, 40, 25]], [[64, 64, 64, 64]], [], [[10, 12, 9, 30]]]
KEYS = ("input_ids", "segment_ids", "input_mask")
ORACLE_CFG = dict(CFG, vocab_size=4096)              # tokens drawn from ~3000 ids, so a word-embedding row sums few token gradients


def _cos(a, b):
    return torch.nn.functional.cosine_similarity(a.float().flatten(), b.float().flatten(), dim=0).item()


def _rel(a, b):
    return ((a.float() - b.float()).norm() / b.float().norm().clamp_min(1e-20)).item()


def _full_state(seed, cfg=CFG):
    from oracle import bert_oracle as O
    sd = {k: v for k, v in O.bf16_representable_params(cfg, seed=seed).items() if k.startswith("bert.")}
    g = torch.Generator().manual_seed(seed + 1)
    sd["classifier.weight"] = (torch.randn(1, cfg["hidden_size"], generator=g) * 0.05).to(bf).float()
    sd["classifier.bias"] = (torch.randn(1, generator=g) * 0.05).to(bf).float()
    return sd


def _prepare(sd, dtype=bf, cfg=CFG, **kw):
    from deeplearningexamples_b200 import swag as W
    return W.prepare_swag_model_and_optimizer(cfg, DEV, C, state_dict=sd, total_steps=kw.pop("total_steps", 100), dtype=dtype, **kw)


def _model(sd, dtype=bf, cfg=CFG):
    return _prepare(sd, dtype, cfg)[0]


# ------------------------------------------------------------------------------------------------------------------------------
# padded model against the fp32 oracle
# ------------------------------------------------------------------------------------------------------------------------------
def test_padded_model_against_fp32_oracle():
    """Scores and the loss against the oracle; gradients of a fixed random projection of the scores.  The cross-entropy's own gradient
    is not compared: an example's dlogits sum to zero over its choices, and its choices share [CLS], [SEP], the context tokens and their
    positions, so the gradients of the embeddings and of the first layers are small differences of C nearly equal sums.  Against the fp32
    oracle they came out at up to 4.5e-2 relative L2 (cosine 0.9990) in bf16, over the 3e-2 bar, while the projection's gradients, which
    run the same backward kernels, keep every bar."""
    from deeplearningexamples_b200 import swag as W
    sd = _full_state(5, ORACLE_CFG)
    batch = W.synthetic_swag_features(4, C, 128, ORACLE_CFG["vocab_size"], seed=6)
    # one full choice row next to ragged ones, its tail filled with real tokens
    n = int(batch["input_mask"][1, 2].sum())
    batch["input_ids"][1, 2, n:] = torch.randint(1000, ORACLE_CFG["vocab_size"], (128 - n,), generator=torch.Generator().manual_seed(7))
    batch["segment_ids"][1, 2, n:] = 1
    batch["input_mask"][1, 2] = 1
    proj = torch.randn(4, C, generator=torch.Generator().manual_seed(8))
    sdo = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    logits_ref = multiple_choice(sdo, ORACLE_CFG, batch["input_ids"], batch["segment_ids"], batch["input_mask"])
    loss_ref = torch.nn.CrossEntropyLoss()(logits_ref, batch["label_ids"])
    (logits_ref * proj).sum().backward()
    model = _model(sd, cfg=ORACLE_CFG).train()
    b = {k: v.to(DEV) for k, v in batch.items()}
    with torch.no_grad():
        loss = model(b["input_ids"], b["segment_ids"], b["input_mask"], b["label_ids"])
    logits = model(b["input_ids"], b["segment_ids"], b["input_mask"])
    (logits.float() * proj.to(DEV)).sum().backward()
    assert logits.shape == (4, C) and logits.dtype == bf and loss.dtype == torch.float32
    lg = logits.detach().float().cpu()
    assert _rel(lg, logits_ref.detach()) < 1e-2, (lg, logits_ref)
    assert abs(loss.item() - loss_ref.item()) < 5e-3 * loss_ref.item(), (loss.item(), loss_ref.item())
    for n, p in model.named_parameters():
        if "pooler" in n:
            assert p.grad is None, n                                                  # frozen, as run_swag.py leaves it untrained
            continue
        want = sdo[n].grad
        if want is None or n.endswith("key.bias") or want.norm() == 0:
            continue
        got = p.grad.float().cpu()
        assert _cos(got, want) > 0.999 and _rel(got, want) < 3e-2, (n, _cos(got, want), _rel(got, want))


# ------------------------------------------------------------------------------------------------------------------------------
# packed against padded
# ------------------------------------------------------------------------------------------------------------------------------
def _examples(choice_lens, seed, vocab=CFG["vocab_size"]):
    """SwagSamples with the given per-choice lengths: [CLS] ... [SEP] rows, segment 1 on each choice's second half."""
    from deeplearningexamples_b200 import packing
    g = torch.Generator().manual_seed(seed)
    out = []
    for e, lens in enumerate(choice_lens):
        ids, segs = [], []
        for n in lens:
            t = torch.randint(1000, vocab, (n,), generator=g)
            t[0], t[-1] = 101, 102
            ids.append(t.numpy())
            segs.append((torch.arange(n) >= n // 2).long().numpy())
        out.append(packing.SwagSample(ids, segs, int(torch.randint(0, C, (1,), generator=g)), e))
    return out


def _packed(row_lens, seed, B=None):
    """A packed SWAG batch whose row r holds examples with the choice lengths row_lens[r], and the examples in order."""
    from deeplearningexamples_b200 import packing
    samples = _examples([ex for r in row_lens for ex in r], seed)
    rows, i = [], 0
    for r in row_lens:
        rows.append(list(range(i, i + len(r))))
        i += len(r)
    return packing.to_swag_batch(samples, rows, B or len(row_lens), S, KPR, C), samples


def _padded_by_group(packed, samples):
    """The padded [G, C, S] batch with one example per group of `packed` (so the pooler and head see the same number of rows): a
    group's example with right-padded choices, and for an empty group C two-token filler rows with label -100."""
    G = packed["label_ids"].shape[0]
    b = {k: torch.zeros(G, C, S, dtype=torch.long) for k in KEYS}
    b["label_ids"] = torch.full((G,), -100, dtype=torch.long)
    for g, e in enumerate(packed.example_index):
        if e < 0:
            b["input_ids"][g, :, :2] = torch.tensor([101, 102])
            b["input_mask"][g, :, :2] = 1
            continue
        s = samples[int(e)]
        for c in range(C):
            n = len(s.input_ids[c])
            b["input_ids"][g, c, :n] = torch.from_numpy(s.input_ids[c])
            b["segment_ids"][g, c, :n] = torch.from_numpy(s.segment_ids[c])
            b["input_mask"][g, c, :n] = 1
        b["label_ids"][g] = s.label
    return b


def _slots(packed):
    """(slot g*C + c, flat positions in the packed batch) of choice c of each example; the slot is also its padded row."""
    am = packed["input_mask"]
    out = []
    for r in range(am.shape[0]):
        for j in range(1, KPR + 1):
            where = torch.nonzero(am[r] == j).squeeze(-1)
            if where.numel():
                out.append((r * KPR + j - 1, r * S + where))
    return out


@pytest.mark.parametrize("cfg", [CFG, WIDE], ids=["small", "wide"])
@pytest.mark.parametrize("dtype", [bf, torch.float32])
def test_packed_eval_logits_equal_padded_logits(dtype, cfg):
    model = _model(_full_state(31, cfg), dtype, cfg).eval()
    packed, samples = _packed(ROW_LENS, seed=32)
    padded = _padded_by_group(packed, samples)
    assert sum(len(c) for c in samples[2].input_ids) == S and bool((packed["input_mask"][2] == 0).all())
    with torch.no_grad():
        l_pad = model(*(padded[k].to(DEV) for k in KEYS))
        model.pack_sequences(KPR)
        l_pk = model(*(packed[k].to(DEV) for k in KEYS))
        model.pack_sequences(0)
    G = len(ROW_LENS) * KPR // C
    assert l_pk.shape == l_pad.shape == (G, C) and l_pk.dtype == l_pad.dtype == dtype
    used = torch.as_tensor(packed.example_index >= 0, device=DEV)
    assert int(used.sum()) == len(samples) == 4
    assert torch.equal(l_pk[used], l_pad[used])                                      # every (example, choice), bit for bit
    assert bool(l_pk.isfinite().all())


def test_packed_512_rows_agree_with_128_token_choice_rows():
    """The benchmark's configuration: examples of 128-token choice rows packed into 512-token rows (k = 16)."""
    from deeplearningexamples_b200 import packing, swag as W
    model = _model(_full_state(35)).eval()
    src = W.synthetic_swag_features(10, C, 128, CFG["vocab_size"], seed=36)
    samples = packing.split_swag_samples(src)
    rows, unplaced = packing.pack(samples, 4, 512, 16 // C, 0)
    assert unplaced == []
    packed = packing.to_swag_batch(samples, rows, 4, 512, 16, C)
    with torch.no_grad():
        l_pad = model(*(src[k].to(DEV) for k in KEYS))
        model.pack_sequences(16)
        l_pk = model(*(packed[k].to(DEV) for k in KEYS))
        model.pack_sequences(0)
    used = packed.example_index >= 0
    got = l_pk[torch.as_tensor(used, device=DEV)].float().cpu()
    want = l_pad.float().cpu()[torch.as_tensor(packed.example_index[used])]
    assert _rel(got, want) < 1e-2, (got, want)


def _swag_step(model, batch):
    """Forward + backward in train mode: (per-group CE terms, mean loss, gradient at the embedding output, parameter gradients).  The
    loss is the model's own labels path; the CE terms come from the same logits without labels."""
    from deeplearningexamples_b200 import ops
    emb = []

    def hook(mod, inp, out):
        if out.requires_grad:
            out.retain_grad()
            emb.append(out)
    h = model.bert.embeddings.register_forward_hook(hook)
    try:
        ops.manual_seed(5)
        b = {k: v.to(DEV) for k, v in batch.items()}
        with torch.no_grad():
            logits = model(b["input_ids"], b["segment_ids"], b["input_mask"])
        rows = torch.nn.CrossEntropyLoss(reduction="none")(logits.float(), b["label_ids"])
        loss = model(b["input_ids"], b["segment_ids"], b["input_mask"], b["label_ids"])
        loss.backward()
        assert torch.equal(loss.detach(), torch.nn.CrossEntropyLoss()(logits.float(), b["label_ids"]))
    finally:
        h.remove()
    grads = {n: p.grad.detach().clone() for n, p in model.named_parameters() if p.grad is not None}
    assert not any("pooler" in n for n in grads)
    model.zero_grad(set_to_none=True)
    return rows.detach(), loss.detach(), emb[-1].grad.detach().reshape(-1, CFG["hidden_size"]).clone(), grads


def test_packed_training_step_equals_padded_step():
    from deeplearningexamples_b200 import swag as W
    model, opt, sched = _prepare(_full_state(41), total_steps=10, learning_rate=1e-2)
    model.train()
    packed, samples = _packed(ROW_LENS, seed=42)
    padded = _padded_by_group(packed, samples)
    rows_pad, l_pad, e_pad, g_pad = _swag_step(model, padded)
    model.pack_sequences(KPR)
    rows_pk, l_pk, e_pk, g_pk = _swag_step(model, packed)
    used = torch.as_tensor(packed.example_index >= 0, device=DEV)
    assert torch.equal(rows_pk[used], rows_pad[used])                             # per-example CE terms
    assert bool((rows_pk[~used] == 0).all())
    assert abs(l_pk.item() - l_pad.item()) <= 1e-5 * abs(l_pad.item())            # the mean, up to fp32 summation order
    example_tokens = torch.zeros(e_pk.shape[0], dtype=torch.bool, device=DEV)
    for slot, fp in _slots(packed):
        n = fp.numel()
        assert torch.equal(e_pk[fp.to(DEV)], e_pad[slot * S:slot * S + n]), slot
        example_tokens[fp.to(DEV)] = True
    assert torch.count_nonzero(e_pk[~example_tokens]) == 0                        # the tail's gradient is exactly zero
    _assert_param_grads_agree({n: g for n, g in g_pk.items() if not n.endswith("key.bias")},
                              {n: g for n, g in g_pad.items() if not n.endswith("key.bias")}, 0.9999, 1e-2)
    # the pooler stays frozen through optimizer steps; the rest trains (the first step runs at lr 0)
    pooler = {n: p.detach().clone() for n, p in model.named_parameters() if "pooler" in n}
    head = model.classifier.weight.detach().clone()
    batch = {k: v.to(DEV) for k, v in packed.items()}
    for _ in range(3):
        W.swag_training_step(model, opt, sched, batch)
    for n, p in model.named_parameters():
        if "pooler" in n:
            assert p.grad is None and torch.equal(p.detach(), pooler[n]), n
    assert not torch.equal(model.classifier.weight.detach(), head)
    model.pack_sequences(0)


def test_padding_free_eval_logits_equal_padded_logits():
    from deeplearningexamples_b200 import swag as W
    model = _model(_full_state(71)).eval()
    b = {k: v.to(DEV) for k, v in W.synthetic_swag_features(6, C, 128, CFG["vocab_size"], seed=72).items()}
    with torch.no_grad():
        want = model(*(b[k] for k in KEYS))
        model.remove_padding(True)
        got = model(*(b[k] for k in KEYS))
        model.remove_padding(False)
    assert bool((b["input_mask"] == 0).any()) and got.shape == (6, C) and torch.equal(got, want)


# ------------------------------------------------------------------------------------------------------------------------------
# CUDA graph
# ------------------------------------------------------------------------------------------------------------------------------
DROP = dict(CFG, hidden_dropout_prob=0.1, attention_probs_dropout_prob=0.1)
TOTAL, WARMUP, LR = 50, 0.1, 1e-4
GRAPH_ROWS = [[[[30, 30, 30, 30], [20, 25, 30, 35]], [[64, 64, 64, 64]], [], [[10, 12, 9, 30]]],
              [[[40, 40, 40, 40]], [[8, 9, 10, 11], [50, 60, 50, 50]], [[2, 3, 4, 5], [60, 60, 60, 60]], [[100, 50, 50, 50]]],
              [[], [[16, 16, 16, 16], [16, 16, 16, 16]], [[64, 64, 64, 60]], [[30, 20, 10, 5]]],
              [[[70, 60, 50, 40]], [], [[5, 5, 5, 5], [5, 5, 5, 5]], [[30, 30, 30, 30], [30, 30, 30, 30]]]]


def _swag_arm(sd):
    """The SWAG training state in the shape test_graph_replay_gpu.py's helpers read (FusedAdam without a loss scaler)."""
    from deeplearningexamples_b200 import ops
    ops.manual_seed(42)                             # same dropout stream ids in both arms
    model, opt, sched = _prepare(sd, cfg=DROP, total_steps=TOTAL, warmup_proportion=WARMUP, learning_rate=LR)
    model.train()
    model.pack_sequences(KPR)
    scaler = types.SimpleNamespace(_scale=torch.ones(1, device=DEV), _growth_tracker=torch.zeros(1, dtype=torch.int32, device=DEV))
    return types.SimpleNamespace(model=model, opt=opt, sched=sched, scaler=scaler, skipped_acc=None,
                                 loss_acc=torch.zeros(1, dtype=torch.float32, device=DEV))


def _step(arm, batch):
    from deeplearningexamples_b200 import swag as W
    W.swag_training_step(arm.model, arm.opt, arm.sched, batch, arm.loss_acc)


def test_replayed_packed_swag_step_matches_eager(seed_log):
    """The whole packed SWAG step (FusedAdam + clip, device-side schedule at the reference's progress global_step / t_total, dropout
    0.1 in the encoder and the head) captured once; before each of three replays a differently packed batch is copied into the static
    buffers and the optimizer's step is set to 0, 1, 2.  Each replay equals eager steps from the same state, which draw the host seeds
    the capture froze, and the lr of each is base * warmup_linear(step / total): exactly 0 at step 0."""
    from deeplearningexamples_b200 import ops, swag as W, training as T
    sd = _full_state(61)
    batches = [{k: v.to(DEV) for k, v in _packed(r, seed=62 + i)[0].items()} for i, r in enumerate(GRAPH_ROWS)]
    g = _swag_arm(sd)
    g.static = {k: v.clone() for k, v in batches[0].items()}
    starts = []

    def one_step():
        starts.append(len(seed_log))
        _step(g, g.static)
    g.graph = T.capture_step_graph(one_step, warmup_iters=3)
    seeds = list(seed_log[starts[-1]:])
    assert len(seeds) == 1 + 3 * DROP["num_hidden_layers"] + 1                # embeddings, 3 per layer, the head
    e = _swag_arm(sd)
    for _ in range(3):
        _step(e, batches[0])
    names = _names(g)
    replay_losses = []
    for i, batch in enumerate(batches[1:]):
        for group in g.opt.param_groups:
            group["step"].fill_(i)
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
        _assert_same_step(got, runs[0], runs[1], names, f"replay {i}")          # lr, loss, step: bitwise
        assert got["found_inf"].item() == 0.0 and got["loss"].isfinite().all()
        want_lr = LR * W.warmup_linear(i / TOTAL, WARMUP)
        assert all(v == pytest.approx(want_lr, rel=1e-6, abs=0.0) for v in got["lr"].tolist()), (i, got["lr"], want_lr)
        if i == 0:
            assert bool((got["lr"] == 0).all()) and all(bool((u == 0).all()) for u in got["updates"])
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


# ------------------------------------------------------------------------------------------------------------------------------
# refusals
# ------------------------------------------------------------------------------------------------------------------------------
def test_pack_sequences_refuses_a_k_that_splits_an_example():
    from deeplearningexamples_b200 import _lib as L
    model = _model(_full_state(81))
    for k in (1, 3, 6, 10):
        with pytest.raises(L.DleError, match="multiple of num_choices"):
            model.pack_sequences(k)
        assert model.bert._pack_per_row == 0
    model.pack_sequences(KPR)
    assert model.bert._pack_per_row == KPR
