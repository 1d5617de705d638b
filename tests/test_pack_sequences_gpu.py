"""GPU: sequence packing (BertPreTrainedModel.pack_sequences).  dle_segment_table against the restatement in
test_pack_sequences_cpu.py; the embedding kernels with explicit positions, bitwise against the NULL path and against fp32; the packed
model against the padded model on the same samples (bitwise where the arithmetic is per row), against the CPU oracle, under a CUDA graph
whose replays read differently packed batches, in LAMB training and under DDP."""
import os
import socket

import numpy as np
import pytest
import torch

from test_graph_replay_gpu import (_assert_same_step, _bench_arm, _bench_step, _clean_state, _counter, _host_seeds, _load,  # noqa: F401
                                   _names, _outcome, _set_counter, _state, seed_log)
from test_pack_sequences_cpu import segment_table_ref
from test_train_packed_gpu import SMALL, _assert_param_grads_agree, _cos, _pretraining_model, _rel_l2, _step

pytestmark = pytest.mark.gpu
bf = torch.bfloat16
DEV = torch.device("cuda", 0)


def _k():
    from deeplearningexamples_b200 import kernels
    return kernels


# ------------------------------------------------------------------------------------------------------------------------------
# segment table
# ------------------------------------------------------------------------------------------------------------------------------
def _random_row(S, k, rng):
    m = int(rng.integers(0, k + 1))
    n = int(rng.integers(m, S + 1)) if m else 0      # real tokens, at least one per sample
    cuts = np.sort(rng.choice(np.arange(1, n), size=m - 1, replace=False)) if m > 1 else np.array([], np.int64)
    lens = np.diff(np.concatenate([[0], cuts, [n]])) if m else []
    return np.concatenate([np.full(int(l), j + 1) for j, l in enumerate(lens)] + [np.zeros(S - n)]).astype(np.int64)


def _run_table(mask, k):
    from deeplearningexamples_b200 import ops
    flag = ops.err_flag(DEV)
    flag.zero_()
    cu, pos, cls = _k().segment_table(torch.as_tensor(mask, device=DEV), k, err_flag=flag)
    return cu.cpu().numpy(), pos.cpu().numpy(), cls.cpu().numpy(), int(flag.item())


@pytest.mark.parametrize("S", [128, 200, 512])
@pytest.mark.parametrize("k", [1, 3, 8])
def test_segment_table_matches_restatement(S, k):
    rng = np.random.default_rng(S * 10 + k)
    rows = [_random_row(S, k, rng) for _ in range(37)]
    rows.append(np.zeros(S, np.int64))                                               # no sample
    full = np.sort(np.concatenate([[1], rng.integers(1, k + 1, S - 1)]))             # exactly k samples, no tail
    full[:k] = np.arange(1, k + 1)
    rows.append(np.sort(full))
    rows.append(np.array([min(j, k) for j in range(1, S + 1)], np.int64) if k > 1 else np.ones(S, np.int64))   # length-1 samples
    rows.append(np.ones(S, np.int64))                                                # one sample fills the row
    mask = np.stack(rows)
    cu, pos, cls, flag = _run_table(mask, k)
    cu_r, pos_r, cls_r, bad = segment_table_ref(mask, k)
    assert bad == [] and flag == 0
    assert np.array_equal(cu, cu_r) and np.array_equal(pos, pos_r) and np.array_equal(cls, cls_r)


@pytest.mark.parametrize("k", [1, 3])
def test_segment_table_flags_malformed_rows_and_stays_in_bounds(k):
    S = 200
    rng = np.random.default_rng(5)
    good = [_random_row(S, k, rng) for _ in range(6)]
    bad_rows = []
    r = np.zeros(S, np.int64); r[:10] = 1; r[10:20] = k + 1; bad_rows.append(r)    # value above k
    r = np.zeros(S, np.int64); r[5] = -3; bad_rows.append(r)                         # negative value
    r = np.zeros(S, np.int64); r[:10] = 1; r[30:40] = 1; bad_rows.append(r)        # non-zero after 0
    r = np.zeros(S, np.int64); r[:10] = 2; bad_rows.append(r)                       # does not start at 1 (skipped number)
    if k > 1:
        r = np.zeros(S, np.int64); r[:10] = 1; r[10:20] = 2; r[20:30] = 1; bad_rows.append(r)     # decrease
    r = np.full(S, 1 << 40, np.int64); bad_rows.append(r)                           # huge value
    for bad_row in bad_rows:
        mask = np.stack(good + [bad_row] + good[:2])
        cu, pos, cls, flag = _run_table(mask, k)
        cu_r, pos_r, cls_r, bad = segment_table_ref(mask, k)
        assert bad == [6] and flag == 1
        assert np.array_equal(cu, cu_r) and np.array_equal(pos, pos_r) and np.array_equal(cls, cls_r)
        assert (np.diff(cu.astype(np.int64)) >= 0).all() and cu[-1] == mask.size
        assert pos.min() >= 0 and pos.max() < S and ((cls == -1) | ((cls >= 0) & (cls < mask.size))).all()


# ------------------------------------------------------------------------------------------------------------------------------
# embedding kernels with explicit positions
# ------------------------------------------------------------------------------------------------------------------------------
def _emb_tables(V, P, H, g):
    t = lambda *s: (torch.randn(*s, generator=g, device=DEV) * 0.5).to(bf)
    return t(V, H), t(P, H), t(2, H), (1 + t(H) * 0.2).to(bf), t(H)


@pytest.mark.parametrize("p_drop", [0.0, 0.1])
@pytest.mark.parametrize("with_seed_dev", [False, True])
@pytest.mark.parametrize("H", [256, 1024])
def test_embedding_with_arange_positions_is_bitwise_the_null_path(p_drop, with_seed_dev, H):
    """B = 2 and distinct token ids: each dword / dpos row sums at most two terms, so the fp32 atomics are order-independent and the
    tables can be compared bit for bit; dtype sums many terms in atomic order and is compared to fp32 rounding."""
    k = _k()
    B, S, V, P = 2, 256, 1024, 512
    g = torch.Generator(device=DEV).manual_seed(H)
    word, pos, typ, gamma, beta = _emb_tables(V, P, H, g)
    ids = torch.randperm(V, generator=g, device=DEV)[:B * S].view(B, S)
    tts = torch.randint(0, 2, (B, S), generator=g, device=DEV)
    dy = torch.randn(B * S, H, generator=g, device=DEV).to(bf)
    sdev = torch.full((1,), 7, dtype=torch.int64, device=DEV) if with_seed_dev else None
    kw = dict(dropout_p=p_drop, seed=99, dropout_stream=4, seed_dev=sdev)
    outs = []
    for position_ids in (None, torch.arange(S, device=DEV).repeat(B, 1)):
        y, z, mean, rstd = k.embed_ln_fwd(ids, tts, word, pos, typ, gamma, beta, position_ids=position_ids, **kw)
        grads = k.embed_ln_bwd(dy, z, mean, rstd, gamma, ids, tts, V, P, 2, position_ids=position_ids, **kw)
        outs.append((y, z, mean, rstd) + tuple(grads))
    (a, b) = outs
    for i, name in enumerate(["y", "z", "mean", "rstd", "dword", "dpos", "dtype", "dgamma", "dbeta"]):
        if name == "dtype":
            torch.testing.assert_close(b[i], a[i], rtol=1e-5, atol=1e-5 * a[i].abs().max().item())
        else:
            assert torch.equal(a[i], b[i]), name
    if p_drop:
        y0 = k.embed_ln_fwd(ids, tts, word, pos, typ, gamma, beta, position_ids=None, **dict(kw, dropout_p=0.0))[0]
        assert not torch.equal(y0, a[0])


def test_embedding_with_arbitrary_positions_vs_fp32():
    from deeplearningexamples_b200 import ops
    k = _k()
    B, S, V, P, H, eps = 4, 200, 512, 512, 768, 1e-12
    g = torch.Generator(device=DEV).manual_seed(3)
    word, pos, typ, gamma, beta = _emb_tables(V, P, H, g)
    ids = torch.randint(0, V, (B, S), generator=g, device=DEV)
    tts = torch.randint(0, 2, (B, S), generator=g, device=DEV)
    position_ids = torch.randint(0, P, (B, S), generator=g, device=DEV)
    dy = torch.randn(B * S, H, generator=g, device=DEV).to(bf)
    flag = ops.err_flag(DEV)
    flag.zero_()
    y, z, mean, rstd = k.embed_ln_fwd(ids, tts, word, pos, typ, gamma, beta, eps=eps, err_flag=flag, position_ids=position_ids)
    dword, dpos, dtyp, dgamma, dbeta = k.embed_ln_bwd(dy, z, mean, rstd, gamma, ids, tts, V, P, 2, position_ids=position_ids)
    assert int(flag.item()) == 0
    W, Pt, Ty, G, Be = (t.float().requires_grad_() for t in (word, pos, typ, gamma, beta))
    zr = W[ids.view(-1)] + Pt[position_ids.view(-1)] + Ty[tts.view(-1)]
    yr = torch.nn.functional.layer_norm(zr, (H,), G, Be, eps)
    (yr * dy.float()).sum().backward()
    assert _rel_l2(y, yr) < 1e-2
    for got, want in ((dword, W.grad), (dpos, Pt.grad), (dtyp, Ty.grad), (dgamma, G.grad), (dbeta, Be.grad)):
        assert _rel_l2(got, want) < 1e-2 and _cos(got, want) > 0.9999
    # a position outside the table is flagged (forward only: the backward trusts the forward's positions)
    position_ids[1, 7] = P
    k.embed_ln_fwd(ids, tts, word, pos, typ, gamma, beta, eps=eps, err_flag=flag, position_ids=position_ids)
    assert int(flag.item()) == 1
    flag.zero_()


# ------------------------------------------------------------------------------------------------------------------------------
# packed model against the padded model on the same samples
# ------------------------------------------------------------------------------------------------------------------------------
def _make_samples(lens, vocab, seed, mlm_fraction=0.15):
    from deeplearningexamples_b200 import packing
    g = torch.Generator().manual_seed(seed)
    out = []
    for n in lens:
        ids = torch.randint(0, vocab, (n,), generator=g)
        ids[0] = 101
        tt = (torch.arange(n) >= n // 2).long()
        lab = torch.full((n,), -1, dtype=torch.long)
        nl = min(max(1, round(mlm_fraction * n)), n - 1)
        where = 1 + torch.randperm(max(n - 1, 0), generator=g)[:nl]
        lab[where] = torch.randint(0, vocab, (where.numel(),), generator=g)
        out.append(packing.Sample(ids.numpy(), tt.numpy(), lab.numpy(), int(torch.randint(0, 2, (1,), generator=g))))
    return out


def _packed_batch(row_lens, S, k, vocab, seed):
    """A packed batch whose row r holds samples of lengths row_lens[r], and the samples in packed order."""
    from deeplearningexamples_b200 import packing
    samples = _make_samples([n for r in row_lens for n in r], vocab, seed)
    rows, i = [], 0
    for r in row_lens:
        rows.append(list(range(i, i + len(r))))
        i += len(r)
    return packing.to_batch(samples, rows, len(row_lens), S, k), samples


def _unpacked_batch(samples, S):
    N = len(samples)
    b = {"input_ids": torch.zeros(N, S, dtype=torch.long), "token_type_ids": torch.zeros(N, S, dtype=torch.long),
         "attention_mask": torch.zeros(N, S, dtype=torch.long), "labels": torch.full((N, S), -1, dtype=torch.long),
         "next_sentence_labels": torch.tensor([s.next_sentence_label for s in samples])}
    for i, s in enumerate(samples):
        n = len(s)
        b["input_ids"][i, :n] = torch.from_numpy(s.input_ids)
        b["token_type_ids"][i, :n] = torch.from_numpy(s.token_type_ids)
        b["attention_mask"][i, :n] = 1
        b["labels"][i, :n] = torch.from_numpy(s.labels)
    return b


def _places(packed, S):
    """For sample i (packed order): (flat positions in the packed batch, flat positions in the unpacked batch, NSP slot)."""
    am, k = packed["attention_mask"], packed["next_sentence_labels"].shape[1]
    out = []
    for r in range(am.shape[0]):
        for j in range(1, k + 1):
            where = torch.nonzero(am[r] == j).squeeze(-1)
            if where.numel():
                i = len(out)
                out.append((r * S + where, i * S + torch.arange(where.numel()), r * k + j - 1))
    return out


ROW_LENS = [[50, 40, 38], [128], [1, 90], [], [70, 30]]       # k samples without tail, a full row, a length-1 sample, an empty row


def test_packed_training_step_equals_padded_step_on_the_same_samples():
    from oracle import bert_oracle as O
    S, k = 128, 3
    sd = O.bf16_representable_params(SMALL, seed=81)
    model = _pretraining_model(SMALL, 0.0, 0.0, sd)
    packed, samples = _packed_batch(ROW_LENS, S, k, SMALL["vocab_size"], seed=82)
    unpacked = _unpacked_batch(samples, S)
    s_pad, n_pad, l_pad, e_pad, g_pad = _step(model, unpacked, seed=9)
    model.pack_sequences(k)
    s_pk, n_pk, l_pk, e_pk, g_pk = _step(model, packed, seed=9)
    model.pack_sequences(0)
    H = e_pk.shape[-1]
    e_pk, e_pad = e_pk.reshape(-1, H), e_pad.reshape(-1, H)
    lab_pk, lab_pad = packed["labels"].reshape(-1), unpacked["labels"].reshape(-1)
    row_pk = torch.cumsum(lab_pk != -1, 0) - 1                 # MLM score row of a labelled flat position
    row_pad = torch.cumsum(lab_pad != -1, 0) - 1
    assert s_pk.shape == s_pad.shape and n_pk.shape == (len(ROW_LENS) * k, 2)
    sample_tokens = torch.zeros(e_pk.shape[0], dtype=torch.bool)
    for i, (fp, fu, slot) in enumerate(_places(packed, S)):
        assert torch.equal(e_pk[fp.cuda()], e_pad[fu.cuda()]), i
        sample_tokens[fp] = True
        lab = lab_pk[fp] != -1
        assert torch.equal(s_pk[row_pk[fp[lab]].cuda()], s_pad[row_pad[fu[lab]].cuda()]), i
        assert torch.equal(n_pk[slot], n_pad[i]), i
    assert torch.count_nonzero(e_pk[~sample_tokens.cuda()]) == 0                # the tail's gradient is exactly zero
    assert abs(l_pk.item() - l_pad.item()) <= 1e-5 * abs(l_pad.item())
    _assert_param_grads_agree(g_pk, g_pad, 0.9999, 1e-2)


def test_packed_inference_equals_padded_inference():
    from oracle import bert_oracle as O
    S, k = 128, 3
    sd = O.bf16_representable_params(SMALL, seed=83)
    model = _pretraining_model(SMALL, 0.0, 0.0, sd).eval()
    packed, samples = _packed_batch(ROW_LENS, S, k, SMALL["vocab_size"], seed=84)
    unpacked = _unpacked_batch(samples, S)
    with torch.no_grad():
        (seq_pad,), pool_pad = model.bert(*(unpacked[key].cuda() for key in ("input_ids", "token_type_ids", "attention_mask")))
        model.pack_sequences(k)
        (seq_pk,), pool_pk = model.bert(*(packed[key].cuda() for key in ("input_ids", "token_type_ids", "attention_mask")))
        model.pack_sequences(0)
    H = seq_pk.shape[-1]
    assert seq_pk.shape == (len(ROW_LENS), S, H) and pool_pk.shape == (len(ROW_LENS) * k, H)
    seq_pk, seq_pad = seq_pk.reshape(-1, H), seq_pad.reshape(-1, H)
    for i, (fp, fu, slot) in enumerate(_places(packed, S)):
        assert torch.equal(seq_pk[fp.cuda()], seq_pad[fu.cuda()]), i
        assert torch.equal(pool_pk[slot], pool_pad[i]), i
    assert bool(torch.isfinite(seq_pk.float()).all()) and bool(torch.isfinite(pool_pk.float()).all())


def test_packed_gradients_vs_cpu_oracle():
    """The bars of test_train_packed_gpu.py::test_pretraining_gradients_vs_cpu_oracle.  A tensor fed by a handful of terms (the pooler and
    NSP head see one row per sample, 7 here) can carry more bf16 rounding than 3e-2 on either route: its relative-L2 bar is
    max(3e-2, 1.25x the padded route's error on the same samples)."""
    from oracle import bert_oracle as O
    S, k = 128, 3
    sd = O.bf16_representable_params(SMALL, seed=61)
    model = _pretraining_model(SMALL, 0.0, 0.0, sd)
    packed, samples = _packed_batch([[60, 40, 28], [128], [100, 1], [77]], S, k, SMALL["vocab_size"], seed=62)
    unpacked = _unpacked_batch(samples, S)
    _, _, _, _, grads_pad = _step(model, unpacked, seed=1)
    model.pack_sequences(k)
    _, _, loss, _, grads = _step(model, packed, seed=1)
    sdo = {key: v.clone().requires_grad_() for key, v in sd.items()}
    loss_ref = O.forward_loss(sdo, SMALL, unpacked)[0]
    loss_ref.backward()
    assert abs(loss.item() - loss_ref.item()) < 1e-2 * loss_ref.item()
    for n, g in grads.items():
        if n.endswith("attention.self.key.bias"):
            continue            # zero in exact arithmetic; both sides hold rounding noise
        want = sdo[n].grad
        assert want is not None and want.norm() > 0, n
        bar = max(3e-2, 1.25 * _rel_l2(grads_pad[n].cpu(), want))
        assert _cos(g.cpu(), want) > 0.999 and _rel_l2(g.cpu(), want) < bar, (n, _cos(g.cpu(), want), _rel_l2(g.cpu(), want), bar)


# ------------------------------------------------------------------------------------------------------------------------------
# CUDA graph, training, DDP
# ------------------------------------------------------------------------------------------------------------------------------
DROP = dict(SMALL, hidden_dropout_prob=0.1, attention_probs_dropout_prob=0.1)
GRAPH_BATCHES = [[[100], [60, 60], [128], [30, 30, 30]],
                 [[40, 40, 40], [], [128], [1, 127]],
                 [[128], [64, 64], [20, 30, 70], []],
                 [[], [90, 9, 1], [10], [100, 28]]]


def test_replayed_packed_step_matches_eager(seed_log):
    """The whole packed step (LAMB, GradScaler, dropout 0.1 at every site) captured once; before each of three replays a differently
    packed batch is copied into the static buffers.  Each replay equals eager steps from the same state, which draw the host seeds
    the capture froze: the packing is read as data, not frozen into the graph."""
    from deeplearningexamples_b200 import training as T
    S, k, P = 128, 3, 20
    batches = [{key: v.to(DEV) for key, v in _packed_batch(r, S, k, DROP["vocab_size"], seed=90 + i)[0].items()}
               for i, r in enumerate(GRAPH_BATCHES)]
    g = _bench_arm(DROP, len(GRAPH_BATCHES[0]), P)
    g.model.pack_sequences(k)
    g.static = {key: v.clone() for key, v in batches[0].items()}
    starts = []

    def one_step():
        starts.append(len(seed_log))
        _bench_step(g, g.static)
    g.graph = T.capture_step_graph(one_step, warmup_iters=3)
    seeds = list(seed_log[starts[-1]:])
    assert len(seeds) == 1 + 3 * DROP["num_hidden_layers"]
    e = _bench_arm(DROP, len(GRAPH_BATCHES[0]), P)
    e.model.pack_sequences(k)
    for _ in range(3):
        _bench_step(e, batches[0])
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
                _bench_step(e, batch)
            runs.append(_outcome(e, pre, [e.loss_acc.clone()]))
        for key in g.static:
            g.static[key].copy_(batch[key])
        _set_counter(c0)
        g.loss_acc.zero_()
        g.graph.replay()
        assert _counter() == c0 + 1
        got = _outcome(g, pre, [g.loss_acc.clone()])
        _assert_same_step(got, runs[0], runs[1], names, f"replay {i}")
        assert got["found_inf"].item() == 0.0 and got["loss"].isfinite().all()
        replay_losses.append(got["loss"].item())
    assert len(set(replay_losses)) == 3, replay_losses
    del g, e


def test_lamb_training_on_packed_rows_reduces_loss_and_is_seed_deterministic():
    """12 LAMB steps with dropout 0.1 on packed rows."""
    from deeplearningexamples_b200 import ops, training
    S, k = 128, 3
    batch = {key: v.cuda() for key, v in _packed_batch([[60, 40, 28], [128], [90, 30], [50, 50]], S, k, SMALL["vocab_size"],
                                                         seed=71)[0].items()}
    runs = []
    for _ in range(2):
        ops.manual_seed(8)                      # before the model is built: its dropout stream ids come from this allocator
        model, opt, scaler, sched, crit, _ = training.prepare_model_and_optimizer(DROP, DEV, learning_rate=2e-3, warmup_proportion=0.1,
                                                                                  max_steps=40, seed=7, init_loss_scale=2 ** 10)
        model.pack_sequences(k)
        losses = []
        for _ in range(12):
            losses.append(training.take_training_step(scaler, model, crit, batch).item())
            training.take_optimizer_step(sched, opt, scaler)
        runs.append(losses)
    ops.check_device_errors()
    assert runs[0][0] == runs[1][0], runs
    assert all(abs(a - b) < 1e-2 * abs(b) for a, b in zip(runs[0], runs[1])), runs
    assert runs[0][-1] < runs[0][0] - 0.3, runs[0]


DDP_CFG = dict(SMALL, max_position_embeddings=128, hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
DDP_ROWS = [[60, 40, 28], [128], [90, 30], []]          # both halves: the same lengths (equal label and sample counts), other tokens


def _ddp_halves():
    halves = [_packed_batch(DDP_ROWS, 128, 3, DDP_CFG["vocab_size"], seed=s)[0] for s in (201, 202)]
    return halves, {key: torch.cat([h[key] for h in halves]) for key in halves[0]}


def _ddp_step(device, distributed, batch):
    from deeplearningexamples_b200 import ops, training as T
    ops.manual_seed(7)
    model, opt, scaler, sched, crit, _ = T.prepare_model_and_optimizer(DDP_CFG, device, learning_rate=1e-3, max_steps=10,
                                                                      warmup_proportion=0.1, distributed=distributed, dtype=torch.float32,
                                                                      seed=11, init_loss_scale=2 ** 10)
    core = model.module if hasattr(model, "module") else model
    core.pack_sequences(3)
    model.train()
    loss = T.take_training_step(scaler, model, crit, {key: v.to(device) for key, v in batch.items()})
    grads = {n: p.grad.detach().float().cpu().clone() for n, p in core.named_parameters() if p.grad is not None}
    T.take_optimizer_step(sched, opt, scaler)
    torch.cuda.synchronize()
    return loss.item(), grads


def _ddp_worker(rank, world, port, out_path):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
    torch.cuda.set_device(rank)
    device = torch.device("cuda", rank)
    dist.init_process_group(backend="nccl", init_method="env://", world_size=world, rank=rank, device_id=device)
    halves, _ = _ddp_halves()
    loss, grads = _ddp_step(device, True, halves[rank])
    losses = [None] * world
    dist.all_gather_object(losses, loss)
    if rank == 0:
        torch.save(dict(losses=losses, grads=grads), out_path)
    dist.barrier()
    dist.destroy_process_group()


def test_two_rank_packed_step_equals_one_rank_step_on_concatenated_batch(tmp_path):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    out = str(tmp_path / "rank0.pt")
    mp.spawn(_ddp_worker, args=(2, port, out), nprocs=2, join=True)
    two = torch.load(out, weights_only=False)
    _, full = _ddp_halves()
    loss, grads = _ddp_step(DEV, False, full)
    assert abs(sum(two["losses"]) / 2 - loss) < 1e-4 * abs(loss)
    for n, g1 in grads.items():
        if n.endswith("key.bias"):
            continue
        assert _rel_l2(two["grads"][n], g1) < 2e-5, (n, _rel_l2(two["grads"][n], g1))


def test_driver_trains_packed_rows_under_cuda_graphs_with_accumulation(tmp_path):
    """run_pretraining.py --pack_sequences 3 --cuda_graphs --gradient_accumulation_steps 2 on the variable-length synthetic source: the
    captured micro-step and full-step graphs replay packed batches, and the run reports samples/s next to rows/s."""
    import json
    from deeplearningexamples_b200 import run_pretraining as rp
    cfg = tmp_path / "cfg.json"
    cfg.write_text(json.dumps(dict(DROP, vocab_size=1021, max_position_embeddings=128)))
    log = tmp_path / "log.json"
    argv = ["--config_file", str(cfg), "--output_dir", str(tmp_path / "out"), "--input_dir", "synthetic", "--do_train", "--fp16",
            "--allreduce_post_accumulation", "--allreduce_post_accumulation_fp16", "--train_batch_size", "8", "--max_seq_length", "128",
            "--max_predictions_per_seq", "20", "--learning_rate", "2e-3", "--warmup_proportion", "0.1", "--json-summary", str(log),
            "--disable_jit_fusions", "--init_loss_scale", "1024", "--max_steps", "100", "--steps_this_run", "6", "--cuda_graphs",
            "--gradient_accumulation_steps", "2", "--skip_checkpoint", "--pack_sequences", "3"]
    rp.cli(argv)
    lines = [json.loads(l)["data"] for l in open(log)]
    final = [d for d in lines if "training_samples_per_second" in d][-1]
    assert 0.0 < final["final_loss"] < 12.0
    # variable-length samples of 32..128 tokens: a packed row holds more than one sample on average
    assert final["training_samples_per_second"] > 1.2 * final["training_sequences_per_second"] > 0
