"""GPU: general distillation.  The relation-KL kernels against the fp32 restatement on the same bf16 operands (attention scores and value
relation, S = 128 and 512, ragged masks with a fully masked row, both token orders), the where rule, identity, determinism and memory;
the cosine-rows kernel; the model-level losses and every student gradient against the fp32 restatement; a captured distillation step
against eager steps."""
import math

import pytest
import torch

from test_distill_cpu import BACKBONE, attention_kl, cosine_loss, distill_losses_fp32, model_states, scores_from_qkv, value_kl

pytestmark = pytest.mark.gpu
bf = torch.bfloat16
DEV = torch.device("cuda", 0)


def _cos(a, b):
    return torch.nn.functional.cosine_similarity(a.float().flatten(), b.float().flatten(), dim=0).item()


def _rel(a, b):
    return ((a.float() - b.float()).norm() / b.float().norm().clamp_min(1e-20)).item()


def _assert_grad(got, ref, what):
    c, r = _cos(got, ref), _rel(got, ref)
    assert c > 0.999 and r < 3e-2, f"{what}: cosine {c:.6f}, rel L2 {r:.3e}"


def _mask(B, S, seed):
    """additive fp32 mask [B, S] with ragged lengths; row 1 is fully masked"""
    g = torch.Generator().manual_seed(seed)
    lens = torch.randint(S // 4, S + 1, (B,), generator=g)
    lens[0] = S
    if B > 1:
        lens[1] = 0
    m = torch.zeros(B, S)
    for b in range(B):
        m[b, lens[b]:] = -10000.0
    return m.to(DEV)


def _qkv(B, S, A, seed, std=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(B * S, 3 * A * 64, generator=g) * std).to(bf).to(DEV)


def _relkl_att(qs, qt, mask, B, S, A, seq_first):
    from deeplearningexamples_b200 import ops
    return ops.RelationKLFn.apply(qs, qt, ("attention", B, S, A, seq_first, mask, mask, 0.125, 0.125))


def _relkl_val(cs, ct, B, S, A, seq_first):
    from deeplearningexamples_b200 import ops
    return ops.RelationKLFn.apply(cs, ct, ("value", B, S, A, seq_first, None, None, 0.125, 0.125))


def _vstates(c, B, S, seq_first):
    """[T, H] attention output in token order -> value states [S, B, H]"""
    return c.view(S, B, -1) if seq_first else c.view(B, S, -1).transpose(0, 1)


# ------------------------------------------------------------------------------------------------------------------------------
# kernels against the fp32 restatement
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("S,B", [(128, 3), (512, 2)])
@pytest.mark.parametrize("seq_first", [False, True])
def test_attention_relkl_against_fp32(S, B, seq_first):
    A = 12
    mask = _mask(B, S, 1)
    qs = _qkv(B, S, A, 2).requires_grad_(True)
    qt = _qkv(B, S, A, 3)
    loss = _relkl_att(qs, qt, mask, B, S, A, seq_first)
    loss.backward()
    ref_in = qs.detach().float().requires_grad_(True)
    ref = attention_kl(scores_from_qkv(ref_in, mask, B, S, A, seq_first), scores_from_qkv(qt.float(), mask, B, S, A, seq_first))
    ref.backward()
    assert abs(loss.item() - ref.item()) <= 5e-3 * abs(ref.item()), (loss.item(), ref.item())
    H = A * 64
    _assert_grad(qs.grad[:, :H], ref_in.grad[:, :H], "dQ")
    _assert_grad(qs.grad[:, H:2 * H], ref_in.grad[:, H:2 * H], "dK")
    assert torch.count_nonzero(qs.grad[:, 2 * H:]) == 0


@pytest.mark.parametrize("S,B", [(128, 3), (512, 2)])
@pytest.mark.parametrize("seq_first", [False, True])
def test_value_relkl_against_fp32(S, B, seq_first):
    A = 12
    g = torch.Generator().manual_seed(7)
    cs = (torch.randn(B * S, A * 64, generator=g) * 0.5).to(bf).to(DEV).requires_grad_(True)
    ct = (torch.randn(B * S, A * 64, generator=g) * 0.5).to(bf).to(DEV)
    loss = _relkl_val(cs, ct, B, S, A, seq_first)
    loss.backward()
    ref_in = cs.detach().float().requires_grad_(True)
    ref = value_kl(_vstates(ref_in, B, S, seq_first), _vstates(ct.float(), B, S, seq_first), A, A, B)
    ref.backward()
    assert abs(loss.item() - ref.item()) <= 5e-3 * abs(ref.item()), (loss.item(), ref.item())
    _assert_grad(cs.grad, ref_in.grad, "d ctx")


def test_where_rule_substitutes_logit_zero_with_zero_gradient():
    """Key 5 of (b 0, head 0) scores about -900 against every query while unmasked: the where rule makes it logit 0, and it gets exactly
    zero gradient in both dK and (through it) nothing else from that column."""
    B, S, A = 2, 128, 12
    H = A * 64
    mask = _mask(B, S, 4)
    qs = _qkv(B, S, A, 5, std=0.3)
    qs[:S, 0] = 30.0                         # every query of b 0, head 0 has a large component on dim 0
    qs[5, H:2 * H] = 0.0
    qs[5, H] = -30.0                         # key 5 of b 0, head 0: q.k/8 ~ -112 for every query
    qt = _qkv(B, S, A, 6, std=0.3)
    qs.requires_grad_(True)
    loss = _relkl_att(qs, qt, mask, B, S, A, False)
    loss.backward()
    scores = scores_from_qkv(qs.detach(), mask, B, S, A, False)
    assert (scores[0, 0, :, 5] <= -100).all() and mask[0, 5] == 0
    ref_in = qs.detach().float().requires_grad_(True)
    ref = attention_kl(scores_from_qkv(ref_in, mask, B, S, A, False), scores_from_qkv(qt.float(), mask, B, S, A, False))
    ref.backward()
    assert abs(loss.item() - ref.item()) <= 5e-3 * abs(ref.item())
    assert torch.count_nonzero(qs.grad[5, H:H + 64]) == 0              # dK of the substituted key: exactly 0
    assert torch.count_nonzero(ref_in.grad[5, H:H + 64]) == 0
    _assert_grad(qs.grad[:, :2 * H], ref_in.grad[:, :2 * H], "dQ|dK")


def test_identical_teacher_gives_exact_zeros():
    B, S, A = 2, 256, 12
    mask = _mask(B, S, 8)
    qs = _qkv(B, S, A, 9).requires_grad_(True)
    loss = _relkl_att(qs, qs.detach().clone(), mask, B, S, A, False)
    loss.backward()
    assert loss.item() == 0.0 and torch.count_nonzero(qs.grad) == 0
    cs = _qkv(B, S, A, 10)[:, :A * 64].contiguous().requires_grad_(True)
    loss = _relkl_val(cs, cs.detach().clone(), B, S, A, True)
    loss.backward()
    assert loss.item() == 0.0 and torch.count_nonzero(cs.grad) == 0


def test_relkl_is_deterministic():
    B, S, A = 2, 512, 12
    mask = _mask(B, S, 11)
    qt = _qkv(B, S, A, 12)
    out = []
    for _ in range(2):
        qs = _qkv(B, S, A, 13).requires_grad_(True)
        loss = _relkl_att(qs, qt, mask, B, S, A, False) + _relkl_val(qs[:, 2 * A * 64:], qt[:, 2 * A * 64:], B, S, A, False)
        loss.backward()
        out.append((loss.detach().clone(), qs.grad.clone()))
    assert torch.equal(out[0][0], out[1][0]) and torch.equal(out[0][1], out[1][1])


def test_memory_at_phase2_shape():
    """fwd + bwd of both KL losses through ops.RelationKLFn at B = 32, S = 512, A = 12.  Beyond the operands, the step holds the
    gradients of the two inputs, each the size of its input (qkv [T, 3H] and ctx [T, H] bf16, 100 MB together; a layer's backward
    consumes them).  Everything else -- lse, partials, the losses -- stays under 64 MB; one fp32 [B, A, S, S] tensor is 402 MB."""
    B, S, A = 32, 512, 12
    H = A * 64
    mask = _mask(B, S, 14)
    qs = _qkv(B, S, A, 15, std=0.5).requires_grad_(True)
    qt = _qkv(B, S, A, 16, std=0.5)
    cs = qs.detach()[:, 2 * H:].contiguous().requires_grad_(True)
    ct = qt[:, 2 * H:]
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    loss = _relkl_att(qs, qt, mask, B, S, A, False) + _relkl_val(cs, ct, B, S, A, False)
    loss.backward()
    torch.cuda.synchronize()
    grads = qs.grad.numel() * qs.grad.element_size() + cs.grad.numel() * cs.grad.element_size()
    extra = torch.cuda.max_memory_allocated() - base - grads
    assert extra < 64 * 2 ** 20, f"{extra / 2 ** 20:.1f} MB beyond the {grads / 2 ** 20:.1f} MB of input gradients"
    assert math.isfinite(loss.item()) and loss.item() > 0


def test_cosine_rows_against_fp32():
    from deeplearningexamples_b200 import ops
    g = torch.Generator().manual_seed(17)
    x = torch.randn(1000, 768, generator=g).to(bf).to(DEV).requires_grad_(True)
    y = (x.detach().float().cpu() + torch.randn(1000, 768, generator=g)).to(bf).to(DEV)
    loss = ops.CosineRowsFn.apply(x, y)
    loss.backward()
    ref_in = x.detach().float().requires_grad_(True)
    ref = cosine_loss(ref_in, y.float(), 768)
    ref.backward()
    assert abs(loss.item() - ref.item()) <= 1e-4 * abs(ref.item())
    _assert_grad(x.grad, ref_in.grad, "d pred")
    loss2 = ops.CosineRowsFn.apply(x, y)
    assert torch.equal(loss.detach(), loss2.detach())


# ------------------------------------------------------------------------------------------------------------------------------
# model level
# ------------------------------------------------------------------------------------------------------------------------------
CFG = dict(hidden_size=768, num_hidden_layers=2, num_attention_heads=12, intermediate_size=3072, vocab_size=1024,
           max_position_embeddings=128, type_vocab_size=2, hidden_act="gelu", initializer_range=0.02,
           hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)


def _params(cfg, seed):
    from oracle import bert_oracle as O
    return {k: v for k, v in O.bf16_representable_params(cfg, seed=seed).items() if k.startswith("bert.") and ".pooler." not in k}


def _batch(B, S, vocab, seed):
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(0, vocab, (B, S), generator=g)
    lens = torch.randint(S // 3, S + 1, (B,), generator=g)
    lens[0] = S
    am = (torch.arange(S)[None, :] < lens[:, None]).long()
    tt = (torch.arange(S)[None, :] >= (lens[:, None] // 2)).long() * am
    return {"input_ids": ids.to(DEV), "token_type_ids": tt.to(DEV), "attention_mask": am.to(DEV)}


def _setup(n_student, mapping, dtype, student_hidden=768, distill=None):
    from deeplearningexamples_b200 import distill as D
    dc = {"distillation": True, "distillation_config": dict(BACKBONE["distillation_config"], student_teacher_layer_mapping=mapping,
                                                            **(distill or {}))}
    s_cfg = dict(CFG, num_hidden_layers=n_student, hidden_size=student_hidden, intermediate_size=4 * student_hidden,
                 num_attention_heads=student_hidden // 64)
    t_sd, s_sd = _params(CFG, 31), _params(s_cfg, 32)
    g = torch.Generator().manual_seed(33)
    p_sd = None
    if student_hidden != CFG["hidden_size"]:
        p_sd = {"fit_dense.weight": (torch.randn(768, student_hidden, generator=g) * 0.05).to(bf).float(),
                "fit_dense.bias": (torch.randn(768, generator=g) * 0.05).to(bf).float()}
    out = D.prepare_distill_models_and_optimizer(s_cfg, CFG, DEV, dc, total_steps=100, dtype=dtype, teacher_state_dict=
                                                 {k[5:]: v for k, v in t_sd.items()}, student_state_dict=s_sd, project_state_dict=p_sd)
    return out, (s_cfg, s_sd, t_sd, p_sd, dc)


def _assert_student_grads(params, ref_sd, n_layers):
    """Every student gradient against the fp32 restatement.  query.bias and value.bias are compared on their own, like every other
    parameter.  key.bias is compared only inside the layer's packed q|k|v bias vector: softmax is invariant to a shift of a query's
    logits, so the key bias gradient is 0 in exact arithmetic apart from the where rule's term (a substituted logit does not shift), and
    on its own it is dominated by the rounding noise of either side."""
    bias = lambda sd, i, get: torch.cat([get(sd[f"bert.encoder.layer.{i}.attention.self.{n}.bias"]) for n in ("query", "key", "value")])  # noqa: E731
    for k, ref in ref_sd.items():
        assert params[k].grad is not None, k
        if k.endswith("attention.self.key.bias"):
            continue
        _assert_grad(params[k].grad, ref.grad, k)
    for i in range(n_layers):
        _assert_grad(bias(params, i, lambda p: p.grad.float()), bias(ref_sd, i, lambda p: p.grad), f"layer {i} q|k|v bias")


def test_query_bias_gradient_carries_the_kl_term():
    """The KL losses reach the q / k biases only through the layer's gradient fold (dle_add_rows_bf16 adds the loss's column sums to
    the bias accumulator).  With the hidden-state loss off, every gradient of the layer comes from the two KL losses: the value loss's
    through the attention backward's own bias sums, the attention loss's only through the fold.  The query bias gradient must then
    equal the restatement's, which it cannot if the fold drops the attention loss's share."""
    from deeplearningexamples_b200 import distill as D
    (student, teacher, project, losses, _o, _s), (s_cfg, s_sd, t_sd, _p, dc) = _setup(1, "last_layer", bf,
                                                                                       distill=dict(use_hidden_states=False))
    student.train(); teacher.train()
    B, S = 4, 128
    batch = _batch(B, S, CFG["vocab_size"], 36)
    att, rep, val = D.distill_losses(student, teacher, project, losses, batch)
    assert rep.item() == 0.0
    (att + val).backward()
    ref_sd = {k: v.to(DEV).requires_grad_(True) for k, v in s_sd.items()}
    s_states = model_states(ref_sd, s_cfg, "bert.", batch["input_ids"], batch["token_type_ids"], batch["attention_mask"])
    with torch.no_grad():
        t_states = model_states({k: v.to(DEV) for k, v in t_sd.items()}, CFG, "bert.", batch["input_ids"], batch["token_type_ids"],
                                batch["attention_mask"])
    r_att, _, r_val = distill_losses_fp32(s_states, t_states, s_cfg, CFG, dc["distillation_config"], B)
    (r_att + r_val).backward()
    k = "bert.encoder.layer.0.attention.self.query.bias"
    got, ref = dict(student.named_parameters())[k].grad, ref_sd[k].grad
    assert ref.norm() > 0
    _assert_grad(got, ref, k)


@pytest.mark.parametrize("dtype", [bf, torch.float32])
@pytest.mark.parametrize("n_student,mapping", [(1, "last_layer"), (2, "last_layer"), (1, "uniform"), (2, "uniform")])
def test_model_losses_and_gradients_against_fp32(n_student, mapping, dtype):
    from deeplearningexamples_b200 import distill as D
    (student, teacher, project, losses, _opt, _sch), (s_cfg, s_sd, t_sd, p_sd, dc) = _setup(n_student, mapping, dtype)
    student.train(); teacher.train()
    B, S = 4, 128
    batch = _batch(B, S, CFG["vocab_size"], 34)
    att, rep, val = D.distill_losses(student, teacher, project, losses, batch)
    (att + rep + val).backward()

    ref_sd = {k: v.to(DEV).requires_grad_(True) for k, v in s_sd.items()}
    cpu_b = {k: v for k, v in batch.items()}
    s_states = model_states(ref_sd, s_cfg, "bert.", cpu_b["input_ids"], cpu_b["token_type_ids"], cpu_b["attention_mask"])
    with torch.no_grad():
        t_states = model_states({k: v.to(DEV) for k, v in t_sd.items()}, CFG, "bert.", cpu_b["input_ids"], cpu_b["token_type_ids"],
                                cpu_b["attention_mask"])
    r_att, r_rep, r_val = distill_losses_fp32(s_states, t_states, s_cfg, CFG, dc["distillation_config"], B)
    (r_att + r_rep + r_val).backward()
    for got, ref, name in ((att, r_att, "att"), (rep, r_rep, "rep"), (val, r_val, "value")):
        assert abs(got.item() - ref.item()) <= 5e-3 * abs(ref.item()), (name, got.item(), ref.item())
    _assert_student_grads(dict(student.named_parameters()), ref_sd, n_student)


def test_model_with_projection_against_fp32():
    """A 512-wide student (8 heads) against the 768-wide teacher: hidden and embedding states only, through Project."""
    from deeplearningexamples_b200 import distill as D
    (student, teacher, project, losses, _o, _s), (s_cfg, s_sd, t_sd, p_sd, dc) = _setup(
        1, "last_layer", bf, student_hidden=512,
        distill=dict(use_attention_scores=False, use_value_states=False, use_embedding_states=True))
    assert project is not None
    student.train(); teacher.train()
    B, S = 2, 128
    batch = _batch(B, S, CFG["vocab_size"], 35)
    att, rep, val = D.distill_losses(student, teacher, project, losses, batch)
    (att + rep + val).backward()
    ref_sd = {k: v.to(DEV).requires_grad_(True) for k, v in s_sd.items()}
    ref_p = [p_sd["fit_dense.weight"].to(DEV).requires_grad_(True), p_sd["fit_dense.bias"].to(DEV).requires_grad_(True)]
    s_states = model_states(ref_sd, s_cfg, "bert.", batch["input_ids"], batch["token_type_ids"], batch["attention_mask"])
    with torch.no_grad():
        t_states = model_states({k: v.to(DEV) for k, v in t_sd.items()}, CFG, "bert.", batch["input_ids"], batch["token_type_ids"],
                                batch["attention_mask"])
    _, r_rep, _ = distill_losses_fp32(s_states, t_states, s_cfg, CFG, dc["distillation_config"], B, project=ref_p)   # + embeddings
    assert att.item() == 0.0 and val.item() == 0.0
    assert abs(rep.item() - r_rep.item()) <= 5e-3 * abs(r_rep.item()), (rep.item(), r_rep.item())
    r_rep.backward()
    _assert_student_grads(dict(student.named_parameters()), ref_sd, 1)
    _assert_grad(project.fit_dense.weight.grad, ref_p[0].grad, "fit_dense.weight")
    _assert_grad(project.fit_dense.bias.grad, ref_p[1].grad, "fit_dense.bias")


# ------------------------------------------------------------------------------------------------------------------------------
# the step under a CUDA graph
# ------------------------------------------------------------------------------------------------------------------------------
def _opt_state(opt):
    """Everything FusedAdam reads or writes for a step, as live tensors in a fixed order: parameters, fp32 masters, moments."""
    ps = [p for g in opt.param_groups for p in g["params"]]
    ms = [p.detach() if m is None else m for p, m in zip(ps, [m for g in opt.param_groups_fp32 for m in g["params"]])]
    return ps, ms, [opt.state[p]["exp_avg"] for p in ps], [opt.state[p]["exp_avg_sq"] for p in ps]


@pytest.mark.parametrize("dropout", [0.0, 0.1])
def test_captured_step_equals_eager(dropout):
    """A captured general_distill_step replays as an eager step does from the same training state, host seeds and device step counter,
    in lockstep (test_graph_replay_gpu.py's protocol): before each replay the eager arm takes the graph arm's parameters, masters and
    moments, so that the fp32 atomics of the bias and split-K weight gradients cannot make the arms drift apart.  Loss terms, lr and
    step (the device dropout counter and the optimizer's step count) bitwise; the updated parameters within 1e-5 relative."""
    from test_graph_replay_gpu import _host_seeds
    from deeplearningexamples_b200 import distill as D, ops, training as T
    global CFG
    saved = CFG
    arms = []
    try:
        CFG = dict(saved, hidden_dropout_prob=dropout, attention_probs_dropout_prob=dropout)
        for _ in range(2):
            ops.manual_seed(5)                   # the same dropout stream ids in both arms
            (student, teacher, project, losses, opt, sch), _ = _setup(1, "last_layer", bf)
            student.train(); teacher.train()
            arms.append((student, teacher, project, losses, opt, sch))
    finally:
        CFG = saved
    seeds = [0x1234567 + 7919 * i for i in range(64)]
    B, S = 4, 128
    batches = [_batch(B, S, 1024, 40 + i) for i in range(5)]
    static = {k: v.clone() for k, v in batches[0].items()}
    g_arm, e_arm = arms
    out = {}

    def step():
        with _host_seeds(seeds):
            out["r"] = D.general_distill_step(*g_arm, static)

    def eager(batch):
        with _host_seeds(seeds):
            return D.general_distill_step(*e_arm, batch)

    ops.step_counter(DEV).fill_(0)
    graph = T.capture_step_graph(step, warmup_iters=2)
    ops.step_counter(DEV).fill_(0)
    for _ in range(2):
        eager(static)
    for i in range(1, 5):
        with torch.no_grad():                    # lockstep: the eager arm starts from the graph arm's state
            for dst, src in zip(_opt_state(e_arm[4]), _opt_state(g_arm[4])):
                for a, b in zip(dst, src):
                    a.copy_(b)
        for gg, ge in zip(g_arm[4].param_groups, e_arm[4].param_groups):
            assert torch.equal(torch.as_tensor(gg["step"]), torch.as_tensor(ge["step"]))
        for k in static:
            static[k].copy_(batches[i][k])
        c = ops.step_counter(DEV).clone()
        graph.replay()
        c_graph = ops.step_counter(DEV).clone()
        ops.step_counter(DEV).copy_(c)
        e = eager(batches[i])
        torch.cuda.synchronize()
        for name, got, ref in zip(("loss", "att", "rep", "value"), out["r"], e):
            assert torch.equal(got, ref), (i, name, got.item(), ref.item())
        lr_g, lr_e = g_arm[4].param_groups[0]["lr"], e_arm[4].param_groups[0]["lr"]
        assert torch.equal(torch.as_tensor(lr_g), torch.as_tensor(lr_e))
        # the step: the device dropout counter each arm leaves behind, and the optimizer's group step counters
        assert torch.equal(c_graph, ops.step_counter(DEV)) and int(c_graph.item()) == int(c.item()) + 2
        for gg, ge in zip(g_arm[4].param_groups, e_arm[4].param_groups):
            assert torch.equal(torch.as_tensor(gg["step"]), torch.as_tensor(ge["step"]))
        assert int(torch.as_tensor(g_arm[4].param_groups[0]["step"]).item()) == 2 + i
        for (n, p), (_, q) in zip(g_arm[0].named_parameters(), e_arm[0].named_parameters()):
            assert _rel(p.detach(), q.detach()) < 1e-5, (i, n)
    assert out["r"][0].item() > 0
