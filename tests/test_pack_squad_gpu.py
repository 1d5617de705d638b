"""GPU: packed SQuAD fine-tuning (BertForQuestionAnswering.pack_sequences(k, per_sample_logits=True)).  The span-logit kernels bit for
bit against the restatement in test_pack_squad_cpu.py; the packed QA model against the padded one on the same features (bitwise where
the arithmetic is per row), against the fp32 CPU oracle run on each feature alone, and as a captured SQuAD step whose replays read
differently packed batches."""
import types

import numpy as np
import pytest
import torch

from test_graph_replay_gpu import (_assert_same_step, _clean_state, _counter, _host_seeds, _names, _outcome, _set_counter,  # noqa: F401
                                   _state, _load, seed_log)
from test_pack_sequences_cpu import segment_table_ref
from test_pack_squad_cpu import FILL, span_grad_ref, span_logits_ref
from test_squad_gpu import CFG

pytestmark = pytest.mark.gpu
bf = torch.bfloat16
DEV = torch.device("cuda", 0)
S, KPR = 384, 3
# k samples without a tail, a full row, a length-1 sample, an empty row
ROW_LENS = [[150, 120, 114], [384], [1, 200], [], [250, 100]]


def _cos(a, b):
    return torch.nn.functional.cosine_similarity(a.float().flatten(), b.float().flatten(), dim=0).item()


def _rel(a, b):
    return ((a.float() - b.float()).norm() / b.float().norm().clamp_min(1e-20)).item()


# ------------------------------------------------------------------------------------------------------------------------------
# kernels
# ------------------------------------------------------------------------------------------------------------------------------
def _mask(row_lens, B):
    m = np.zeros((B, S), np.int64)
    for r, lens in enumerate(row_lens):
        off = 0
        for j, n in enumerate(lens, 1):
            m[r, off:off + n] = j
            off += n
    return m


@pytest.mark.parametrize("dtype", [bf, torch.float32])
def test_span_kernels_match_restatement_bit_for_bit(dtype):
    from deeplearningexamples_b200 import kernels as K, ops
    B = 7
    mask = _mask(ROW_LENS + [[10, 10]], B)
    mask[5, 20:30] = 1                                          # malformed (non-zero after 0): one tail segment, every slot fill
    flag = ops.err_flag(DEV)
    flag.zero_()
    cu, _, _ = K.segment_table(torch.as_tensor(mask, device=DEV), KPR, err_flag=flag)
    assert int(flag.item()) == 1
    flag.zero_()
    cu_r, _, _, bad = segment_table_ref(mask, KPR)
    assert bad == [5] and np.array_equal(cu.cpu().numpy(), cu_r)
    g = torch.Generator(device=DEV).manual_seed(1)
    wide = (torch.randn(B * S, 4, generator=g, device=DEV) * 5).to(dtype)
    logits = wide[:, 1:3]                                       # row stride 4
    start, end = K.span_logits_unpack(logits, cu, B, S, KPR, FILL)
    s_r, e_r = span_logits_ref(logits.cpu(), cu_r, B, S, KPR, FILL)
    assert start.dtype == dtype and torch.equal(start.cpu(), s_r) and torch.equal(end.cpu(), e_r)
    assert (start[5 * KPR:6 * KPR] == torch.tensor(FILL, dtype=dtype)).all()
    if dtype == bf:
        assert torch.tensor(FILL, dtype=bf).item() == -9984.0
    ds = (torch.randn(B * KPR, S, generator=g, device=DEV) * 3).to(dtype)
    de = (torch.randn(B * KPR, S, generator=g, device=DEV) * 3).to(dtype)
    d = K.span_logits_pack_grad(ds, de, cu, B, S, KPR)
    d_r = span_grad_ref(ds.cpu(), de.cpu(), cu_r, B, S, KPR)
    assert d.dtype == dtype and torch.equal(d.cpu(), d_r)
    tail = torch.as_tensor(mask == 0).reshape(-1) | torch.as_tensor(np.isin(np.arange(B * S) // S, bad))
    assert torch.count_nonzero(d.cpu()[tail]) == 0 and torch.count_nonzero(d.cpu()[~tail]) > 0
    ops.check_device_errors()


# ------------------------------------------------------------------------------------------------------------------------------
# packed QA model against the padded QA model on the same features
# ------------------------------------------------------------------------------------------------------------------------------
def _full_state(seed):
    from oracle import bert_oracle as O
    sd = O.bf16_representable_params(CFG, seed=seed)
    g = torch.Generator().manual_seed(seed + 1)
    full = {k: v for k, v in sd.items() if k.startswith("bert.")}
    full["qa_outputs.weight"] = (torch.randn(2, CFG["hidden_size"], generator=g) * 0.05).to(bf).float()
    full["qa_outputs.bias"] = (torch.randn(2, generator=g) * 0.05).to(bf).float()
    return sd, full


def _features(lens, seed):
    from deeplearningexamples_b200 import packing
    g = torch.Generator().manual_seed(seed)
    out = []
    for i, n in enumerate(lens):
        ids = torch.randint(0, CFG["vocab_size"], (n,), generator=g)
        ids[0] = 101
        seg = (torch.arange(n) >= max(1, n // 4)).long()
        a = int(torch.randint(0, n, (1,), generator=g))
        b = a + int(torch.randint(0, n - a, (1,), generator=g))
        out.append(packing.SquadSample(ids.numpy(), seg.numpy(), a, b, i))
    return out


def _packed(row_lens, seed, B=None):
    """A packed SQuAD batch whose row r holds features of lengths row_lens[r] (B rows, the rest empty), and the features in order."""
    from deeplearningexamples_b200 import packing
    feats = _features([n for r in row_lens for n in r], seed)
    rows, i = [], 0
    for r in row_lens:
        rows.append(list(range(i, i + len(r))))
        i += len(r)
    return packing.to_squad_batch(feats, rows, B or len(row_lens), S, KPR), feats


def _padded(feats):
    N = len(feats)
    b = {"input_ids": torch.zeros(N, S, dtype=torch.long), "segment_ids": torch.zeros(N, S, dtype=torch.long),
         "input_mask": torch.zeros(N, S, dtype=torch.long),
         "start_positions": torch.tensor([f.start_position for f in feats]), "end_positions": torch.tensor([f.end_position for f in feats])}
    for i, f in enumerate(feats):
        n = len(f)
        b["input_ids"][i, :n] = torch.from_numpy(f.input_ids)
        b["segment_ids"][i, :n] = torch.from_numpy(f.segment_ids)
        b["input_mask"][i, :n] = 1
    return b


def _slots(packed):
    """(slot, length, flat positions in the packed batch) of each feature, in order."""
    am = packed["input_mask"]
    out = []
    for r in range(am.shape[0]):
        for j in range(1, KPR + 1):
            where = torch.nonzero(am[r] == j).squeeze(-1)
            if where.numel():
                out.append((r * KPR + j - 1, where.numel(), r * S + where))
    return out


def _model(full, dtype=bf, cfg=CFG):
    from deeplearningexamples_b200 import squad as SQ
    model, opt, sched = SQ.prepare_squad_model_and_optimizer(cfg, DEV, state_dict=full, total_steps=100, dtype=dtype)
    return model


@pytest.mark.parametrize("dtype", [bf, torch.float32])
def test_packed_eval_logits_equal_padded_logits(dtype):
    """Same number of rows on both routes (the packed batch's extra rows are empty), so the QA head's GEMM has one shape."""
    _, full = _full_state(31)
    model = _model(full, dtype).eval()
    packed, feats = _packed(ROW_LENS, seed=32, B=8)
    padded = _padded(feats)
    assert padded["input_ids"].shape[0] == 8
    keys = ("input_ids", "segment_ids", "input_mask")
    with torch.no_grad():
        s_pad, e_pad = model(*(padded[k].to(DEV) for k in keys))
        model.pack_sequences(KPR, per_sample_logits=True)
        s_pk, e_pk = model(*(packed[k].to(DEV) for k in keys))
        model.pack_sequences(0)
    assert s_pk.shape == e_pk.shape == (8 * KPR, S) and s_pk.dtype == s_pad.dtype
    fill = torch.tensor(FILL, dtype=s_pk.dtype, device=DEV)
    used = torch.zeros(8 * KPR, S, dtype=torch.bool, device=DEV)
    for i, (slot, n, _) in enumerate(_slots(packed)):
        assert torch.equal(s_pk[slot, :n], s_pad[i, :n]) and torch.equal(e_pk[slot, :n], e_pad[i, :n]), i
        used[slot, :n] = True
    assert bool((s_pk[~used] == fill).all()) and bool((e_pk[~used] == fill).all())


def _qa_step(model, batch, mask_padding):
    """Forward + backward in train mode: (per-slot losses, mean loss, gradient at the embedding output, parameter gradients).  With
    mask_padding the logits at masked positions are set to FILL first (the padded route's logits as the packed loss sees them)."""
    from deeplearningexamples_b200 import ops, squad as SQ
    emb = []

    def hook(mod, inp, out):
        out.retain_grad()
        emb.append(out)
    h = model.bert.embeddings.register_forward_hook(hook)
    try:
        ops.manual_seed(5)
        b = {k: v.to(DEV) for k, v in batch.items()}
        s, e = model(b["input_ids"], b["segment_ids"], b["input_mask"])
        if mask_padding:
            keep = b["input_mask"] != 0
            s = torch.where(keep, s, torch.tensor(FILL, dtype=s.dtype, device=DEV))
            e = torch.where(keep, e, torch.tensor(FILL, dtype=e.dtype, device=DEV))
        ce = torch.nn.CrossEntropyLoss(ignore_index=S, reduction="none")
        rows = (ce(s.float(), b["start_positions"].clamp(0, S)) + ce(e.float(), b["end_positions"].clamp(0, S))) / 2
        loss = SQ.squad_loss(s, e, b["start_positions"], b["end_positions"])
        loss.backward()
    finally:
        h.remove()
    grads = {n: p.grad.detach().clone() for n, p in model.named_parameters() if p.grad is not None}
    model.zero_grad(set_to_none=True)
    return rows.detach(), loss.detach(), emb[0].grad.detach().reshape(-1, CFG["hidden_size"]).clone(), grads


# analytically zero gradients (both sides are rounding noise): key biases (softmax shift invariance), the QA bias and the bias of the
# last LayerNorm in front of the linear head (every row of d(loss)/d(logits) sums to zero)
ZERO_GRADS = ("qa_outputs.bias", "bert.encoder.layer.%d.output.LayerNorm.bias" % (CFG["num_hidden_layers"] - 1))


def _analytically_zero(name):
    return name.endswith("key.bias") or name in ZERO_GRADS


def test_packed_training_step_equals_padded_step_with_masked_logits():
    _, full = _full_state(41)
    model = _model(full).train()
    packed, feats = _packed(ROW_LENS, seed=42, B=8)
    rows_pad, l_pad, e_pad, g_pad = _qa_step(model, _padded(feats), mask_padding=True)
    model.pack_sequences(KPR, per_sample_logits=True)
    rows_pk, l_pk, e_pk, g_pk = _qa_step(model, packed, mask_padding=False)
    model.pack_sequences(0)
    sample_tokens = torch.zeros(e_pk.shape[0], dtype=torch.bool, device=DEV)
    for i, (slot, n, fp) in enumerate(_slots(packed)):
        assert torch.equal(rows_pk[slot], rows_pad[i]), i
        assert torch.equal(e_pk[fp.to(DEV)], e_pad[i * S:i * S + n]), i
        sample_tokens[fp.to(DEV)] = True
    assert torch.count_nonzero(e_pk[~sample_tokens]) == 0                     # the tail's gradient is exactly zero
    assert abs(l_pk.item() - l_pad.item()) <= 1e-5 * abs(l_pad.item())
    assert g_pk.keys() == g_pad.keys() and not any("pooler" in n for n in g_pk)
    for n in g_pad:
        if not _analytically_zero(n):
            assert _cos(g_pk[n], g_pad[n]) > 0.9999, (n, _cos(g_pk[n], g_pad[n]))


def test_packed_loss_and_gradients_vs_fp32_oracle_per_feature():
    """Each feature alone, unpadded at its own length, through the fp32 oracle with the QA head and the reference's span loss
    (run_squad.py:1073-1079): the bars of test_squad_gpu.py."""
    from oracle import bert_oracle as O
    sd, full = _full_state(51)
    model = _model(full).train()
    packed, feats = _packed([[150, 120, 114], [384], [1, 200], [250, 100]], seed=52)
    model.pack_sequences(KPR, per_sample_logits=True)
    _, loss, _, grads = _qa_step(model, packed, mask_padding=False)
    sdo = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    w = full["qa_outputs.weight"].clone().requires_grad_(True)
    b_ = full["qa_outputs.bias"].clone().requires_grad_(True)
    ls, le = [], []
    for f in feats:
        n = len(f)
        ids, seg = torch.from_numpy(f.input_ids).view(1, n), torch.from_numpy(f.segment_ids).view(1, n)
        seq, _ = O.bert_model(sdo, CFG, ids, seg, torch.ones(1, n, dtype=torch.long))
        logits = torch.nn.functional.linear(seq, w, b_)
        lf = torch.nn.CrossEntropyLoss(ignore_index=n)
        ls.append(lf(logits[..., 0], torch.tensor([f.start_position]).clamp(0, n)))
        le.append(lf(logits[..., 1], torch.tensor([f.end_position]).clamp(0, n)))
    loss_ref = (torch.stack(ls).mean() + torch.stack(le).mean()) / 2
    loss_ref.backward()
    assert abs(loss.item() - loss_ref.item()) < 5e-3 * loss_ref.item(), (loss.item(), loss_ref.item())
    for k, p in model.named_parameters():
        if "pooler" in k:
            assert k not in grads
            continue
        want = w.grad if k == "qa_outputs.weight" else b_.grad if k == "qa_outputs.bias" else sdo[k].grad
        if want is None or _analytically_zero(k):
            continue
        got = grads[k].float().cpu()
        assert _cos(got, want) > 0.999 and _rel(got, want) < 3e-2, (k, _cos(got, want), _rel(got, want))


# ------------------------------------------------------------------------------------------------------------------------------
# CUDA graph
# ------------------------------------------------------------------------------------------------------------------------------
DROP = dict(CFG, hidden_dropout_prob=0.1, attention_probs_dropout_prob=0.1)
GRAPH_ROWS = [[[300], [150, 150], [384], [100, 100, 100]],
              [[120, 120, 120], [], [384], [1, 383]],
              [[384], [192, 192], [50, 80, 200], []],
              [[], [250, 90, 1], [30], [300, 84]]]


def _squad_arm(full):
    """The SQuAD training state in the shape test_graph_replay_gpu.py's helpers read.  FusedAdam runs without a loss scaler: the
    scaler fields are constants."""
    from deeplearningexamples_b200 import ops, squad as SQ
    ops.manual_seed(42)                             # same dropout stream ids in both arms
    model, opt, sched = SQ.prepare_squad_model_and_optimizer(DROP, DEV, state_dict=full, total_steps=50, learning_rate=1e-4)
    model.train()
    model.pack_sequences(KPR, per_sample_logits=True)
    scaler = types.SimpleNamespace(_scale=torch.ones(1, device=DEV), _growth_tracker=torch.zeros(1, dtype=torch.int32, device=DEV))
    return types.SimpleNamespace(model=model, opt=opt, sched=sched, scaler=scaler, skipped_acc=None,
                                 loss_acc=torch.zeros(1, dtype=torch.float32, device=DEV))


def _squad_step(arm, batch):
    from deeplearningexamples_b200 import squad as SQ
    SQ.squad_training_step(arm.model, arm.opt, arm.sched, batch, arm.loss_acc)


def test_replayed_packed_squad_step_matches_eager(seed_log):
    """The whole packed SQuAD step (FusedAdam + clip, device-side schedule, dropout 0.1) captured once; before each of three replays a
    differently packed batch is copied into the static buffers.  Each replay equals eager steps from the same state, which draw the
    host seeds the capture froze."""
    from deeplearningexamples_b200 import ops, training as T
    _, full = _full_state(61)
    batches = [{k: v.to(DEV) for k, v in _packed(r, seed=62 + i)[0].items()} for i, r in enumerate(GRAPH_ROWS)]
    g = _squad_arm(full)
    g.static = {k: v.clone() for k, v in batches[0].items()}
    starts = []

    def one_step():
        starts.append(len(seed_log))
        _squad_step(g, g.static)
    g.graph = T.capture_step_graph(one_step, warmup_iters=3)
    seeds = list(seed_log[starts[-1]:])
    assert len(seeds) == 1 + 3 * DROP["num_hidden_layers"]
    e = _squad_arm(full)
    for _ in range(3):
        _squad_step(e, batches[0])
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
                _squad_step(e, batch)
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
    assert len(set(replay_losses)) == 3, replay_losses
    ops.check_device_errors()
    del g, e
