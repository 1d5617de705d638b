"""GPU: a replayed CUDA graph of the training step computes the step the eager code computes.

While a step is captured, Python runs once and its decisions are frozen into every replay: the host dropout seeds, whether the LAMB
device table is re-patched, whether a gradient is assigned or accumulated, whether an fp32 parameter is recast to bf16.  Each test here
runs two arms built from the same seeds: arm G is captured and then only replayed, arm E only ever runs eagerly.  Before each compared
step G's whole training state is copied into E in place, and the shared device step counter is set to the same value for both.  Then

  * the forward, hence the loss, and the scalars of the step (lr, group step, loss scale, growth tracker, found_inf, skipped steps) must
    be bitwise equal;
  * gradients and parameter updates (post - pre) are not bitwise reproducible (split-K weight gradients, column sums and the embedding
    tables sum with fp32 atomics): each tensor must lie within 4x the relative L2 distance of two eager runs from the same state, with
    a floor of 1e-4.  One pair of eager runs can underestimate the spread of those sums against a replay, whose launch timing differs
    (at the benchmarked widths the q/k/v bias updates, whose gradients largely cancel, came out 1.6e-5 to 4.6e-5 apart while two eager
    runs agreed within 1e-5); a replay that misses or repeats work moves updates by 1e-2 or more.

The eager step itself is anchored to the CPU LAMB oracle on the real parameter list.
"""
import copy
import itertools
import json
import types

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
bf = torch.bfloat16
DEV = torch.device("cuda", 0)

SMALL = dict(hidden_size=256, num_hidden_layers=2, num_attention_heads=4, intermediate_size=1024, vocab_size=1024,
             max_position_embeddings=512, type_vocab_size=2, hidden_act="gelu", initializer_range=0.02,
             hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
# the benchmarked widths (BERT-large, bench.py), two layers: the real GEMM tile and split-K choices
WIDE = dict(SMALL, hidden_size=1024, num_attention_heads=16, intermediate_size=4096, vocab_size=30528)
FLOOR = 1e-4


@pytest.fixture(autouse=True)
def _clean_state():
    from deeplearningexamples_b200 import ops
    yield
    ops.step_counter(DEV).zero_()
    ops._w16_cache.clear()
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------------------------------------
# training state of an arm: snapshot, in-place load, outcome of a step
# ------------------------------------------------------------------------------------------------------------------------------
def _params(arm):
    return [p for g in arm.opt.param_groups for p in g["params"]]


def _names(arm):
    by_id = {id(p): n for n, p in arm.model.named_parameters()}
    return [by_id[id(p)] for p in _params(arm)]


def _masters(arm):
    """The fp32 tensors LAMB updates: the master copies of bf16 parameters, fp32 parameters themselves."""
    ms = [m for g in arm.opt.param_groups_fp32 for m in g["params"]]
    return [p.detach() if m is None else m for p, m in zip(_params(arm), ms)]


def _state(arm):
    """Clones of everything a training step reads or writes."""
    ps, opt = _params(arm), arm.opt
    return dict(params=[p.detach().clone() for p in ps], masters=[m.clone() for m in _masters(arm)],
                exp_avg=[opt.state[p]["exp_avg"].clone() for p in ps], exp_avg_sq=[opt.state[p]["exp_avg_sq"].clone() for p in ps],
                step=[g["step"].clone() for g in opt.param_groups], scale=arm.scaler._scale.clone(),
                growth=arm.scaler._growth_tracker.clone(), grads=[None if p.grad is None else p.grad.clone() for p in ps],
                skipped=None if arm.skipped_acc is None else arm.skipped_acc.clone())


def _load(arm, st):
    """Copy a state into `arm` in place.  Parameters through p.copy_() so that their version counters move and cached bf16 copies of
    fp32 parameters are invalidated (p.data.copy_ would not move them)."""
    ps, opt = _params(arm), arm.opt
    with torch.no_grad():
        for p, v in zip(ps, st["params"]):
            p.copy_(v)
        for m, v in zip(_masters(arm), st["masters"]):
            m.copy_(v)
        for p, a, b in zip(ps, st["exp_avg"], st["exp_avg_sq"]):
            opt.state[p]["exp_avg"].copy_(a)
            opt.state[p]["exp_avg_sq"].copy_(b)
        for g, s in zip(opt.param_groups, st["step"]):
            g["step"].copy_(s)
        arm.scaler._scale.copy_(st["scale"])
        arm.scaler._growth_tracker.copy_(st["growth"])
        for p, gr in zip(ps, st["grads"]):
            if gr is None:
                p.grad = None
            elif p.grad is None:
                p.grad = gr.clone()
            else:
                p.grad.copy_(gr)
        if arm.skipped_acc is not None:
            arm.skipped_acc.copy_(st["skipped"])


def _outcome(arm, pre, losses, grads=None):
    """What a step produced, relative to the state `pre` it started from."""
    opt = arm.opt
    return dict(loss=torch.stack([l.reshape(()) for l in losses]), lr=torch.stack([g["lr"].reshape(()).clone() for g in opt.param_groups]),
                step=torch.cat([g["step"].clone() for g in opt.param_groups]), scale=arm.scaler._scale.clone(),
                growth=arm.scaler._growth_tracker.clone(), found_inf=opt._found_inf.clone(),
                skipped=None if arm.skipped_acc is None else arm.skipped_acc.clone(),
                updates=[m.float() - m0.float() for m, m0 in zip(_masters(arm), pre["masters"])], grads=grads)


def _rel(a, b):
    a, b = a.float(), b.float()
    d, n = (a - b).norm().item(), b.norm().item()
    return d / n if n > 0 else d


def _assert_same_step(got, e1, e2, names, what):
    """got: the replay; e1, e2: two eager runs from the same state."""
    for k in ("loss", "lr", "step", "scale", "growth", "found_inf", "skipped"):
        if e1[k] is None:
            continue
        assert torch.equal(e1[k], e2[k]), f"{what}: two eager runs disagree on {k}: {e1[k]} vs {e2[k]}"
        assert torch.equal(got[k], e1[k]), f"{what}: {k} of the replay {got[k].tolist()} != eager {e1[k].tolist()}"
    for k in ("updates", "grads"):
        if e1[k] is None:
            continue
        bad = []
        for n, g, a, b in zip(names, got[k], e1[k], e2[k]):
            bar = max(4 * _rel(b, a), FLOOR)
            r = _rel(g, a)
            if not r <= bar:
                bad.append((n, r, bar))
        assert not bad, f"{what}: {k} of the replay off the eager ones (name, rel L2, bar): {bad[:8]} ({len(bad)} tensors)"


def _set_counter(c):
    from deeplearningexamples_b200 import ops
    ops.step_counter(DEV).fill_(c)


def _counter():
    from deeplearningexamples_b200 import ops
    return int(ops.step_counter(DEV).item())


# ------------------------------------------------------------------------------------------------------------------------------
# the benchmarked step: training.prepare_model_and_optimizer + take_training_step + take_optimizer_step (bench.py)
# ------------------------------------------------------------------------------------------------------------------------------
def _bench_arm(cfg, B, P, seed=42):
    from deeplearningexamples_b200 import ops, training as T
    ops.manual_seed(seed)                      # same dropout stream ids in both arms
    model, opt, scaler, sched, crit, config = T.prepare_model_and_optimizer(cfg, DEV, seed=seed, static_masked_count=B * P)
    model.train()
    return types.SimpleNamespace(model=model, opt=opt, scaler=scaler, sched=sched, crit=crit, skipped_acc=None,
                                 loss_acc=torch.zeros(1, dtype=torch.float32, device=DEV), vocab=config.vocab_size)


def _bench_step(arm, batch):
    from deeplearningexamples_b200 import training as T
    T.take_training_step(arm.scaler, arm.model, arm.crit, batch, arm.loss_acc)
    T.take_optimizer_step(arm.sched, arm.opt, arm.scaler)


def _batches(n, B, S, vocab, P, seed):
    from deeplearningexamples_b200 import training as T
    return [T.synthetic_batch(B, S, vocab, P, seed=seed + i, full_mask=(i % 2 == 0), device=DEV) for i in range(n)]


def _capture_bench(cfg, B, S, P, seed_log=None):
    """Arms G (captured, as bench.py does: 3 eager warm-ups then capture) and E (3 eager warm-ups: lazy LAMB moments exist)."""
    from deeplearningexamples_b200 import training as T
    g = _bench_arm(cfg, B, P)
    batches = _batches(4, B, S, g.vocab, P, seed=7)
    g.static = {k: v.clone() for k, v in batches[0].items()}
    starts = []

    def one_step():
        starts.append(len(seed_log) if seed_log is not None else 0)
        _bench_step(g, g.static)
    g.graph = T.capture_step_graph(one_step, warmup_iters=3)
    g.captured_seeds = None if seed_log is None else list(seed_log[starts[-1]:])
    e = _bench_arm(cfg, B, P)
    for _ in range(3):
        _bench_step(e, batches[0])
    return g, e, batches[1:]


def _lockstep_bench(g, e, batch, seeds=None):
    """One replay on G and two eager steps on E from G's state; E draws `seeds` (the captured host seeds) when given."""
    from deeplearningexamples_b200 import ops
    pre, c0 = _state(g), _counter()
    runs = []
    for _ in range(2):
        _load(e, pre)
        _set_counter(c0)
        e.loss_acc.zero_()
        with _host_seeds(seeds):
            _bench_step(e, batch)
        runs.append(_outcome(e, pre, [e.loss_acc.clone()]))
    for k in g.static:
        g.static[k].copy_(batch[k])
    _set_counter(c0)
    g.loss_acc.zero_()
    g.graph.replay()
    assert _counter() == c0 + 1
    got = _outcome(g, pre, [g.loss_acc.clone()])
    return got, runs, pre, c0


class _host_seeds:
    """Within the block, ops.next_seed returns `seeds` in order (nothing changes when seeds is None)."""

    def __init__(self, seeds):
        self.seeds = seeds

    def __enter__(self):
        from deeplearningexamples_b200 import ops
        self.real = ops.next_seed
        if self.seeds is not None:
            it = iter(self.seeds)
            ops.next_seed = lambda: next(it)

    def __exit__(self, *exc):
        from deeplearningexamples_b200 import ops
        ops.next_seed = self.real


@pytest.mark.parametrize("cfg,B,S,P", [(SMALL, 4, 128, 20), (WIDE, 8, 512, 80)], ids=["small", "wide"])
def test_replayed_bench_step_matches_eager(cfg, B, S, P):
    """(a) bf16, dropout 0: three replays of the benchmarked step on different batches, each against eager steps from the same state."""
    from oracle import lamb_oracle as LO
    g, e, batches = _capture_bench(cfg, B, S, P)
    names = _names(g)
    for i, batch in enumerate(batches):
        got, (e1, e2), pre, _ = _lockstep_bench(g, e, batch)
        _assert_same_step(got, e1, e2, names, f"replay {i}")
        assert got["found_inf"].item() == 0.0 and got["loss"].isfinite().all()
        # the replayed schedule follows the optimizer's step, not the step it was captured at
        step = int(pre["step"][0].item())
        assert got["lr"][0].item() == pytest.approx(LO.poly_warmup_lr(step, 7038, 0.2843, 6e-3), rel=1e-6), (i, step)
        # the bf16 parameters are the rounding of the updated masters
        assert all(torch.equal(p.detach(), m.to(bf)) for p, m in zip(_params(g), _masters(g)))
    del g, e


@pytest.fixture
def seed_log(monkeypatch):
    """The host seeds the dropout call sites draw, in order."""
    from deeplearningexamples_b200 import ops
    drawn, real = [], ops.next_seed

    def logged():
        s = real()
        drawn.append(s)
        return s
    monkeypatch.setattr(ops, "next_seed", logged)
    return drawn


def test_replayed_step_with_dropout_matches_eager(seed_log):
    """(b) dropout 0.1 on every site: E draws the host seeds the capture froze, in order (embedding, then attention, attention-output
    and output dropout of each layer), at the counter value of the replay.  The loss must be bitwise equal.  Control: with one site's
    seed changed, E's loss differs."""
    cfg = dict(SMALL, hidden_dropout_prob=0.1, attention_probs_dropout_prob=0.1)
    B, S, P = 4, 128, 20
    g, e, batches = _capture_bench(cfg, B, S, P, seed_log=seed_log)
    seeds = g.captured_seeds
    assert len(seeds) == 1 + 3 * cfg["num_hidden_layers"] and len(set(seeds)) == len(seeds)
    names = _names(g)
    for i, batch in enumerate(batches):
        got, (e1, e2), pre, c0 = _lockstep_bench(g, e, batch, seeds=seeds)
        _assert_same_step(got, e1, e2, names, f"replay {i}")
        if i == 0:
            # embedding, layer-0 attention, layer-0 attention output, last layer's output: each site's mask reaches the loss
            for site in (0, 1, 2, len(seeds) - 1):
                wrong = list(seeds)
                wrong[site] ^= 0x5DEECE66D
                _load(e, pre)
                _set_counter(c0)
                e.loss_acc.zero_()
                with _host_seeds(wrong):
                    _bench_step(e, batch)
                assert not torch.equal(e.loss_acc, e1["loss"].reshape(1)), f"the loss does not see dropout site {site}"
    del g, e


def test_eager_step_matches_lamb_oracle():
    """(c) one eager step of the benchmarked setup against the CPU LAMB oracle on the real parameter list: the two groups (no_decay
    by name), the tied decoder weight (one parameter), the packed q|k|v views (three parameters over one storage), the scaled
    gradients as the step saw them, and lr from the PolyWarmUp schedule.  Masters and moments at the bars of test_lamb_gpu.py, and
    each bf16 parameter equal to bf16(master)."""
    from oracle import lamb_oracle as LO
    B, S, P = 4, 128, 20
    e = _bench_arm(SMALL, B, P)
    batches = _batches(3, B, S, e.vocab, P, seed=11)
    for b in batches[:2]:                                  # non-zero moments, step 2
        _bench_step(e, b)
    named = dict(e.model.named_parameters())
    no_decay = ["bias", "gamma", "beta", "LayerNorm"]
    g0, g1 = e.opt.param_groups
    assert {id(p) for p in g0["params"]} == {id(p) for n, p in named.items() if not any(nd in n for nd in no_decay)}
    assert {id(p) for p in g1["params"]} == {id(p) for n, p in named.items() if any(nd in n for nd in no_decay)}
    assert g0["weight_decay"] == 0.01 and g1["weight_decay"] == 0.0
    assert e.model.cls.predictions.decoder.weight is e.model.bert.embeddings.word_embeddings.weight
    att = e.model.bert.encoder.layer[0].attention.self
    assert att.key.weight.data_ptr() == att.query.weight.data_ptr() + att.query.weight.numel() * 2

    from deeplearningexamples_b200 import training as T
    T.take_training_step(e.scaler, e.model, e.crit, batches[2], e.loss_acc)
    scale = e.scaler._scale.item()
    og = []
    for group, g32 in zip(e.opt.param_groups, e.opt.param_groups_fp32):
        live = [(p, m) for p, m in zip(group["params"], g32["params"]) if p.grad is not None]
        assert len(live) == len(group["params"])
        step = int(group["step"].item())
        og.append(dict(params=[m.cpu().numpy().copy() for _, m in live], grads=[p.grad.float().cpu().numpy() for p, _ in live],
                       exp_avg=[e.opt.state[p]["exp_avg"].cpu().numpy().copy() for p, _ in live],
                       exp_avg_sq=[e.opt.state[p]["exp_avg_sq"].cpu().numpy().copy() for p, _ in live],
                       lr=LO.poly_warmup_lr(step, 7038, 0.2843, 6e-3), betas=group["betas"], eps=group["eps"],
                       weight_decay=group["weight_decay"], step=step, bias_correction=True, grad_averaging=True))
    T.take_optimizer_step(e.sched, e.opt, e.scaler)
    r = LO.lamb_step(og, scale=scale)
    assert not r["found_inf"] and e.opt._found_inf.item() == 0.0
    assert e.opt._global_grad_norm.item() == pytest.approx(r["global_grad_norm"], rel=1e-5)
    for group, g32, ogrp in zip(e.opt.param_groups, e.opt.param_groups_fp32, og):
        assert group["step"].item() == ogrp["step"] == 3
        assert group["lr"].item() == pytest.approx(ogrp["lr"], rel=1e-6)
        for i, (p, m) in enumerate(zip(group["params"], g32["params"])):
            st = e.opt.state[p]
            np.testing.assert_allclose(st["exp_avg"].cpu().numpy(), ogrp["exp_avg"][i], rtol=1e-5, atol=1e-9)
            np.testing.assert_allclose(st["exp_avg_sq"].cpu().numpy(), ogrp["exp_avg_sq"][i], rtol=1e-5, atol=1e-12)
            np.testing.assert_allclose(m.cpu().numpy(), ogrp["params"][i], rtol=1e-5, atol=1e-7)
            assert torch.equal(p.detach(), m.to(bf))


# ------------------------------------------------------------------------------------------------------------------------------
# the driver's graphs: run_pretraining.capture_training_graphs
# ------------------------------------------------------------------------------------------------------------------------------
DRIVER_CFG = dict(attention_probs_dropout_prob=0.0, hidden_act="gelu", hidden_dropout_prob=0.0, hidden_size=256, initializer_range=0.02,
                  intermediate_size=1024, max_position_embeddings=128, num_attention_heads=4, num_hidden_layers=2, type_vocab_size=2,
                  vocab_size=1021)


def _driver_args(tmp_path, accum, fp32_params):
    """Driver arguments as setup_training leaves them: the per-micro-step batch, and in fp32-parameter mode (--fp16 in a single
    process) the model kept in fp32; bf16 mode is what --allreduce_post_accumulation_fp16 gives a DDP rank."""
    from deeplearningexamples_b200 import run_pretraining as rp
    cfg = tmp_path / "cfg.json"
    cfg.write_text(json.dumps(DRIVER_CFG))
    argv = ["--config_file", str(cfg), "--output_dir", str(tmp_path / "out"), "--do_train", "--fp16", "--cuda_graphs",
            "--train_batch_size", str(2 * accum), "--gradient_accumulation_steps", str(accum), "--max_seq_length", "128",
            "--max_predictions_per_seq", "10", "--learning_rate", "2e-3", "--warmup_proportion", "0.1", "--max_steps", "30",
            "--init_loss_scale", "1024"]
    if not fp32_params:
        argv += ["--allreduce_post_accumulation", "--allreduce_post_accumulation_fp16"]
    args = rp.parse_arguments(argv)
    args.local_rank = -1
    args.train_batch_size //= accum
    return args


def _driver_arm(args, seed=42):
    from deeplearningexamples_b200 import ops, run_pretraining as rp
    torch.manual_seed(seed)
    ops.manual_seed(seed)
    model, opt, scaler, sched, _, _, crit, _, config = rp.prepare_model_and_optimizer(args, DEV, sequence_output_is_dense=True)
    model.train()
    return types.SimpleNamespace(model=model, opt=opt, scaler=scaler, sched=sched, crit=crit, args=args, vocab=config.vocab_size,
                                 loss_acc=torch.zeros(1, dtype=torch.float32, device=DEV),
                                 skipped_acc=torch.zeros(1, dtype=torch.float32, device=DEV))


def _driver_arms(args):
    """G: capture_training_graphs on a static batch, then the statistics rewound as main() does.  E: the eager driver (zero_grad with
    set_to_none=True), one eager optimizer step so that its LAMB moments exist."""
    from deeplearningexamples_b200 import run_pretraining as rp
    g = _driver_arm(args)
    k = args.gradient_accumulation_steps
    batches = _batches(1 + 3 * k, args.train_batch_size, args.max_seq_length, g.vocab, args.max_predictions_per_seq, seed=21)
    g.static = {n: v.clone() for n, v in batches[0].items()}
    g.full, g.accum = rp.capture_training_graphs(args, g.model, g.opt, g.scaler, g.sched, g.crit, g.static, g.loss_acc, g.skipped_acc)
    assert (g.accum is None) == (k == 1)
    g.loss_acc.zero_()
    g.skipped_acc.zero_()
    e = _driver_arm(copy.copy(args))
    e.args.cuda_graphs = False
    _eager_driver_step(e, batches[:k])
    return g, e, [batches[1 + i * k:1 + (i + 1) * k] for i in range(3)]


def _eager_driver_step(arm, micro):
    """The eager driver loop over one optimizer step's micro-batches; returns (losses, gradients before the last micro-step)."""
    from deeplearningexamples_b200 import run_pretraining as rp
    losses, grads = [], None
    for i, b in enumerate(micro):
        if i == len(micro) - 1:
            grads = [None if p.grad is None else p.grad.clone() for p in _params(arm)]
        arm.loss_acc.zero_()
        rp.take_training_step(arm.args, arm.scaler, arm.model, arm.crit, b, arm.loss_acc)
        losses.append(arm.loss_acc.clone())
    rp.take_optimizer_step(arm.args, arm.sched, arm.opt, arm.scaler, arm.skipped_acc)
    return losses, grads


def _w16_want(model):
    """cache key of ops.w16 -> the bf16 copy of the parameter's current value.  The encoder layers cast the q|k|v parameters as one
    packed block, cached under the query parameter."""
    qkv = {id(p) for m in model.modules() if hasattr(m, "_packed") and hasattr(m, "query")
           for lin in (m.query, m.key, m.value) for p in (lin.weight, lin.bias)}
    nsp = {id(p) for p in model.cls.seq_relationship.parameters()}      # the [B, 2] NSP head is torch's nn.Linear in fp32
    want = {(id(p), tuple(p.shape)): p.detach().to(bf) for p in model.parameters() if id(p) not in qkv | nsp}
    for m in model.modules():
        if hasattr(m, "_packed") and hasattr(m, "query"):
            w, b = m._packed()
            want[(id(m.query.weight), tuple(w.shape))] = w.to(bf)
            want[(id(m.query.bias), tuple(b.shape))] = b.to(bf)
    return want


def _assert_w16_cache(want, what):
    from deeplearningexamples_b200 import ops
    keys = [k for k in ops._w16_cache if k in want]
    assert len(keys) == len(want), f"{what}: only {len(keys)} of {len(want)} parameters have a cached bf16 copy"
    stale = [k for k in keys if not torch.equal(ops._w16_cache[k][1], want[k])]
    assert not stale, f"{what}: {len(stale)} of {len(keys)} cached bf16 copies are not bf16 of the weights the step read"


def _replay_driver_step(g, micro, fp32_params):
    """The driver loop under --cuda_graphs over one optimizer step; returns (losses, gradients before the full-step replay)."""
    losses, grads = [], None
    for i, b in enumerate(micro):
        last = i == len(micro) - 1
        for n in g.static:
            g.static[n].copy_(b[n])
        if last:
            grads = [None if p.grad is None else p.grad.clone() for p in _params(g)]
        want = _w16_want(g.model) if fp32_params else None
        g.loss_acc.zero_()
        (g.full if last else g.accum).replay()
        losses.append(g.loss_acc.clone())
        if fp32_params:                # every replay read bf16 copies of the weights as they were when it started
            _assert_w16_cache(want, f"after {'the full-step' if last else 'micro-step'} replay {i}")
    return losses, grads


@pytest.mark.parametrize("fp32_params", [False, True], ids=["bf16", "fp32_params"])
@pytest.mark.parametrize("accum", [2, 3])
def test_driver_gradient_accumulation_replay_matches_eager(tmp_path, accum, fp32_params):
    """(e) --cuda_graphs with --gradient_accumulation_steps k: per optimizer step, k-1 micro-step replays and one full-step replay
    against the eager driver over the same micro-batches.  Each micro-step's loss bitwise, the accumulated gradient buffers before the
    full-step replay and the updates after it within the eager-noise bar, the buffers zero afterwards.  In fp32-parameter mode every
    replay must also have read bf16 copies of the current fp32 weights.  Control: a micro-step at the weights before the previous
    update gives a different loss, so the lr is large enough for stale weights to show."""
    args = _driver_args(tmp_path, accum, fp32_params)
    g, e, steps = _driver_arms(args)
    assert all(p.dtype == (torch.float32 if fp32_params else bf) for p in _params(g))
    names = _names(g)
    prev = None
    for s, micro in enumerate(steps):
        pre, c0 = _state(g), _counter()
        assert all(gr is not None and gr.count_nonzero().item() == 0 for gr in pre["grads"])
        runs = []
        for _ in range(2):
            _load(e, pre)
            _set_counter(c0)
            losses, grads = _eager_driver_step(e, micro)
            runs.append(_outcome(e, pre, losses, grads))
        _set_counter(c0)
        losses, grads = _replay_driver_step(g, micro, fp32_params)
        assert _counter() == c0 + accum
        got = _outcome(g, pre, losses, grads)
        _assert_same_step(got, runs[0], runs[1], names, f"optimizer step {s}")
        assert got["found_inf"].item() == 0.0 and got["skipped"].item() == 0.0
        assert all(p.grad is not None and p.grad.count_nonzero().item() == 0 for p in _params(g)), "gradient buffers not zeroed"
        if prev is not None:                               # control: the previous step's weights give another loss
            _load(e, prev)
            _set_counter(c0)
            e.loss_acc.zero_()
            from deeplearningexamples_b200 import run_pretraining as rp
            rp.take_training_step(e.args, e.scaler, e.model, e.crit, micro[0], e.loss_acc)
            assert not torch.equal(e.loss_acc, runs[0]["loss"][0].reshape(1)), "stale weights would not change the loss"
        prev = pre
    del g, e


def test_driver_overflow_skip_under_replay(tmp_path):
    """(d) the overflow path inside the full-step graph: with the loss scale at 2^127 the scaled gradients overflow, so the replay
    must leave parameters, masters, moments and group step bitwise unchanged, set found_inf, halve the scale exactly and count one
    skipped step.  With the scale put back, the next replay steps normally and matches the eager driver."""
    args = _driver_args(tmp_path, 1, fp32_params=False)
    g, e, steps = _driver_arms(args)
    names = _names(g)
    scale0 = g.scaler._scale.clone()
    g.scaler._scale.fill_(2.0 ** 127)
    pre = _state(g)
    _replay_driver_step(g, steps[0], False)
    assert g.opt._found_inf.item() == 1.0
    assert g.scaler._scale.item() == 2.0 ** 126 and g.scaler._growth_tracker.item() == 0
    assert g.skipped_acc.item() == pre["skipped"].item() + 1
    post = _state(g)
    for k in ("params", "masters", "exp_avg", "exp_avg_sq", "step"):
        same = [torch.equal(a, b) for a, b in zip(pre[k], post[k])]
        assert all(same), f"{k} changed on a skipped step: {[n for n, ok in zip(names, same) if not ok][:8]}"
    g.scaler._scale.copy_(scale0)
    pre, c0 = _state(g), _counter()
    runs = []
    for _ in range(2):
        _load(e, pre)
        _set_counter(c0)
        losses, grads = _eager_driver_step(e, steps[1])
        runs.append(_outcome(e, pre, losses))
    _set_counter(c0)
    losses, _ = _replay_driver_step(g, steps[1], False)
    got = _outcome(g, pre, losses)
    _assert_same_step(got, runs[0], runs[1], names, "the replay after the skipped one")
    assert got["found_inf"].item() == 0.0 and got["step"][0].item() == pre["step"][0].item() + 1
    del g, e
