"""Numerics of the fused attention kernels (csrc/attention_sm90.cu): fp64 references, error yardsticks, bars, and proof that the bars
have teeth.

The bars come from an error model, not from measurements.  A kernel whose output is correct to bf16 rounding has an L2 error about
equal to that of rounding the exact result (ratio ~1); one extra bf16 rounding of P on the way adds an error of the same size (ratio
~sqrt(2)).  So the forward is held to 1.25x the rounding of the exact ctx, and the backward to 1.5x a yardstick that rounds exactly
what the kernels round (P, dS and the stored dq / dk / dv) and does everything else in fp64.  The yardstick has to round the stored
gradients too: the final rounding of dV is as large as the rounding of P it follows, and without it the correct simulation's dV
error is 1.4x to 2.6x the yardstick's across the families below.

The tests here run on the CPU.  tiled_forward_sim restates attn_fwd_kernel's algorithm in fp32 -- 64-key tiles in the log2 domain,
running max and sum, P as bf16 hi + lo parts, one final drop_scale / l -- and backward_sim restates the dK/dV and dQ kernels.  The
correct simulations must clear every bar on every input family, and each mutant (one plausible slip in the kernel) must fail one.
tests/test_attention_numerics_gpu.py holds the kernels to the same bars on the H100 with these functions."""
import functools
import math

import numpy as np
import pytest
import torch

from test_attention_wgmma_gpu import _thresh15, reference_keep

bf = torch.bfloat16
HD = 64
LOG2E32 = float(np.float32(1.4426950408889634))        # the kernels' fp32 constants
LN2_32 = float(np.float32(0.6931471805599453))
SCALE_LOG2 = float(np.float32(0.125) * np.float32(LOG2E32))

FWD_RATIO_BAR = 1.25
BWD_RATIO_BAR = 1.5
LSE_ABS, LSE_ULPS = 5e-5, 4.0

FAMILIES = ("std", "sharp3", "sharp5", "spike_early", "spike_late", "rising")


# ------------------------------------------------------------------------------------------------
# layouts: qkv [T, 3H] with token (b, s) at row b*S + s, or s*B + b with seq_first (the reference's [S, B, *] layer convention)
# ------------------------------------------------------------------------------------------------
def split_qkv(qkv, B, S, A, seq_first=False):
    """qkv [T, 3H] -> q, k, v [B, A, S, 64]"""
    x = qkv.reshape(S, B, 3, A, HD).transpose(0, 1) if seq_first else qkv.reshape(B, S, 3, A, HD)
    return [x[:, :, i].permute(0, 2, 1, 3) for i in range(3)]


def split_rows(t, B, S, A, seq_first=False):
    """[T, H] -> [B, A, S, 64]"""
    x = t.reshape(S, B, A, HD).transpose(0, 1) if seq_first else t.reshape(B, S, A, HD)
    return x.permute(0, 2, 1, 3)


def merge_rows(t, seq_first=False):
    """[B, A, S, 64] -> [T, H]"""
    B, A, S, _ = t.shape
    x = t.permute(0, 2, 1, 3)
    if seq_first:
        x = x.transpose(0, 1)
    return x.reshape(B * S, A * HD)


def drop_scale(p):
    """the kernels' 1/(1-p): p quantised to 1/32768 (attn_drop_params), in fp32"""
    t15 = _thresh15(p) if p > 0 else 0
    return float(np.float32(1.0) / (np.float32(1.0) - np.float32(t15) / np.float32(32768.0))) if t15 else 1.0


def keep_mask(B, S, A, p, seed, stream, device="cpu"):
    """the kernels' dropout keep bits, bool [B, A, S, S] (or None when p = 0)"""
    return torch.from_numpy(reference_keep(B, S, A, p, seed, stream)).to(device) if p > 0 else None


def _bf16(x):
    return x.to(bf).to(x.dtype)


def _fma32(a, b, c):
    """fmaf(a, b, c) on fp32 tensors: the fp64 product of two fp32 values is exact, so this rounds (as good as) once"""
    return (a.double() * b + (c.double() if torch.is_tensor(c) else c)).float()


# ------------------------------------------------------------------------------------------------
# fp64 reference and yardstick
# ------------------------------------------------------------------------------------------------
def attention_ref64(qkv, mask, B, S, A, seq_first=False, keep=None, p=0.0, dctx=None):
    """BertSelfAttention (modeling.py: scores / sqrt(d) + mask, softmax, dropout, @ V) in fp64 on the given bf16 inputs.  keep: bool
    [B, A, S, S] dropout keep mask, rescaled by the kernels' drop_scale(p).  Returns ctx [T, H], lse [B, A, S] and, given dctx,
    dqkv [T, 3H] (else None), all fp64."""
    q, k, v = (t.double() for t in split_qkv(qkv, B, S, A, seq_first))
    s = q @ k.transpose(-1, -2) / 8
    if mask is not None:
        s = s + mask.double().view(B, 1, 1, S)
    lse = torch.logsumexp(s, -1)
    P = torch.exp(s - lse[..., None])
    dsc = drop_scale(p)
    Pt = P * keep * dsc if keep is not None else P
    ctx = merge_rows(Pt @ v, seq_first)
    if dctx is None:
        return ctx, lse, None
    do = split_rows(dctx, B, S, A, seq_first).double()
    dp = do @ v.transpose(-1, -2)
    if keep is not None:
        dp = dp * keep * dsc
    dS = P * (dp - (P * dp).sum(-1, keepdim=True)) / 8
    grads = (dS @ k, dS.transpose(-1, -2) @ q, Pt.transpose(-1, -2) @ do)
    return ctx, lse, torch.cat([merge_rows(g, seq_first) for g in grads], 1)


def backward_yardstick(qkv, mask, ctx, dctx, lse64, B, S, A, seq_first=False, keep=None, p=0.0):
    """The backward at the precision the kernels claim: fp64, except that P and dS are rounded to bf16 before their products (the
    kernels' pack_bf16 of P and dS), delta is taken from the saved bf16 ctx, and dq / dk / dv are rounded to bf16 as the kernels
    store them.  lse64: the fp64 reference's lse."""
    q, k, v = (t.double() for t in split_qkv(qkv, B, S, A, seq_first))
    s = q @ k.transpose(-1, -2) / 8
    if mask is not None:
        s = s + mask.double().view(B, 1, 1, S)
    P = _bf16(torch.exp(s - lse64[..., None]))
    dsc = drop_scale(p)
    Pt = P * keep if keep is not None else P
    do = split_rows(dctx, B, S, A, seq_first).double()
    delta = (do * split_rows(ctx, B, S, A, seq_first).double()).sum(-1, keepdim=True)
    dS = _bf16((Pt * (do @ v.transpose(-1, -2)) * dsc - P * delta) / 8)
    grads = (dS @ k, dS.transpose(-1, -2) @ q, Pt.transpose(-1, -2) @ do * dsc)
    return torch.cat([merge_rows(_bf16(g), seq_first) for g in grads], 1)


# ------------------------------------------------------------------------------------------------
# bars
# ------------------------------------------------------------------------------------------------
def _ratio(num, den):
    if den == 0.0:
        return 0.0 if num == 0.0 else math.inf
    return num / den


def fwd_ratio(ctx, ref):
    """||ctx - ref|| / ||bf16(ref) - ref||: ~1 for ctx correct to bf16 rounding, ~sqrt(2) with one more bf16 rounding of P"""
    ref = ref.double()
    return _ratio((ctx.double() - ref).norm().item(), (_bf16(ref) - ref).norm().item())


def _ulp(x, mant_bits):
    _, e = torch.frexp(x.abs())
    return torch.where(x == 0, torch.zeros_like(x), torch.ldexp(torch.ones_like(x), e - mant_bits - 1))


def fwd_elem_excess(ctx, ref, floor):
    """max over elements of |ctx - ref| / (2 bf16 ulps of |ref| + floor), floor from elem_floor.  Passes at <= 1."""
    ref = ref.double()
    return ((ctx.double() - ref).abs() / (2.0 * _ulp(ref, 7) + floor)).max().item()


def lse_excess(lse, lse64):
    """max |lse - lse64| / (5e-5 + 4 fp32 ulps of lse64).  Passes at <= 1."""
    lse64 = lse64.double()
    return ((lse.double() - lse64).abs() / (LSE_ABS + LSE_ULPS * _ulp(lse64, 23))).max().item()


def rel_err(x, ref):
    return _ratio((x.double() - ref).norm().item(), ref.norm().item())


def bwd_ratios(dqkv, yard, ref, H):
    """relative L2 error of each of dq, dk, dv over the yardstick's.  Passes at <= BWD_RATIO_BAR."""
    out = {}
    for i, name in enumerate("qkv"):
        sl = slice(i * H, (i + 1) * H)
        out["d" + name] = _ratio(rel_err(dqkv[:, sl], ref[:, sl]), rel_err(yard[:, sl], ref[:, sl]))
    return out


def elem_floor(qkv, mask, B, S, A, seq_first=False):
    """The absolute term of the per-element bound, per (b, h), shaped like ctx [T, H]: 2^-14 max|v| (P carried to ~16 bits).  A row
    whose every key is masked adds ln2 * ulp_fp32(|mask| * log2e) * max|v|: each of its scores fmaf(s, scale*log2e, mask*log2e) is
    rounded at the ulp of the mask term (2^-10 for -10000), which moves every P by up to that much relatively -- the cost of the
    reference's additive -10000 in fp32, in which the reference itself adds it."""
    vmax = split_qkv(qkv, B, S, A, seq_first)[2].double().abs().amax(dim=(-1, -2))            # [B, A]
    rel = torch.full((B, 1), 2.0 ** -14, dtype=torch.float64, device=qkv.device)
    if mask is not None:
        t = (mask.float() * LOG2E32).double().abs().amin(-1, keepdim=True)                     # 0 unless every key is masked
        rel = rel + LN2_32 * _ulp(t, 23)
    return merge_rows((rel * vmax)[:, :, None, None].expand(B, A, S, HD), seq_first)


def forward_scores(ctx, lse, ref_ctx, ref_lse, floor):
    return dict(fwd_ratio=fwd_ratio(ctx, ref_ctx), elem=fwd_elem_excess(ctx, ref_ctx, floor), lse=lse_excess(lse, ref_lse))


BARS = dict(fwd_ratio=FWD_RATIO_BAR, elem=1.0, lse=1.0, dq=BWD_RATIO_BAR, dk=BWD_RATIO_BAR, dv=BWD_RATIO_BAR)


def over_bars(sc):
    """the bars a score dict fails"""
    return [k for k, v in sc.items() if not v <= BARS[k]]


# ------------------------------------------------------------------------------------------------
# input families
# ------------------------------------------------------------------------------------------------
def edge_lens(S):
    """one row per key-tile / query-tile edge length up to S, and an all-padding row"""
    return sorted({n for n in (1, 63, 64, 65, 127, 128, 129, S - 1, S) if n <= S}) + [0]


def lens_mask(lens, S, device="cpu"):
    keep = (torch.arange(S).unsqueeze(0) < torch.as_tensor(lens).unsqueeze(1)).float()
    return ((1.0 - keep) * -10000.0).to(device)


def family_qkv(family, B, S, A, lens=None, seed=0, device="cpu"):
    """bf16 qkv [B*S, 3H] (batch-first) of one input family:
      std, sharp3, sharp5: N(0, sigma^2) with sigma 1, 3, 5 -- score std sigma^2;
      spike_early / spike_late: sigma 1, plus one key per (b, h) in the first / last valid 64-key tile whose score is 8 above the rest
        (q feature 0 = 4, k feature 0 = 16 there and 0 elsewhere), so the row max is set in that tile;
      rising: sigma 1, q feature 0 = 4 and k feature 0 rising from -16 to 16 with the key index, so scores gain 16 over the
        sequence, the row max grows from tile to tile and every tile rescales."""
    g = torch.Generator().manual_seed(seed)
    sigma = {"sharp3": 3.0, "sharp5": 5.0}.get(family, 1.0)
    x = torch.randn(B, S, 3, A, HD, generator=g) * sigma
    if family in ("spike_early", "spike_late", "rising"):
        x[:, :, 0, :, 0] = 4.0
        if family == "rising":
            x[:, :, 1, :, 0] = torch.linspace(-16.0, 16.0, S).view(1, S, 1)
        else:
            x[:, :, 1, :, 0] = 0.0
            for b in range(B):
                n = int(lens[b]) if lens is not None and int(lens[b]) > 0 else S
                lo = 0 if family == "spike_early" else (n - 1) // 64 * 64
                idx = torch.randint(lo, min(lo + 64, n), (A,), generator=g)
                x[b, idx, 1, torch.arange(A), 0] = 16.0
    return x.reshape(B * S, 3 * A * HD).to(bf).to(device)


def rand_dctx(T, H, seed, device="cpu"):
    return torch.randn(T, H, generator=torch.Generator().manual_seed(seed)).to(bf).to(device)


# ------------------------------------------------------------------------------------------------
# fp32 restatements of the kernels, with mutants
# ------------------------------------------------------------------------------------------------
FWD_MUTANTS = {
    "a_no_lo": "the lo part of P dropped (P to V as bf16 only)",
    "b_no_o_rescale": "o not rescaled when the row max grows",
    "c_no_l_rescale": "l not rescaled when the row max grows",
    "d_mask_not_log2e": "the additive mask not multiplied by log2(e)",
    "e_lse_log2": "lse stored in log2 units",
}
BWD_MUTANTS = {
    "f_pdrop_delta": "P~ (dropped) in the -P*delta term of dS",
    "g_dk_no_scale": "the softmax scale missing from dK",
}


def tiled_forward_sim(qkv, mask, B, S, A, seq_first=False, keep=None, p=0.0, mutant=None):
    """attn_fwd_kernel's algorithm in fp32: per 64-key tile, t = fmaf(s, scale*log2e, mask*log2e), running max m and sum l (rescaled
    by ex2(m_old - m_new)), P = ex2(t - m) to the MMA as bf16 hi + lo parts (AND the keep mask), l summed before dropout, then ctx =
    bf16(o * drop_scale / l) and lse = (m + log2 l) * ln2.  Returns ctx bf16 [T, H], lse fp32 [B, A, S]."""
    q, k, v = (t.float() for t in split_qkv(qkv, B, S, A, seq_first))
    if mask is None:
        mk = torch.zeros(B, S, device=qkv.device)
    else:
        mk = mask.float() if mutant == "d_mask_not_log2e" else mask.float() * LOG2E32
    m = torch.full((B, A, S), -math.inf, device=qkv.device)
    l = torch.zeros(B, A, S, device=qkv.device)
    o = torch.zeros(B, A, S, HD, device=qkv.device)
    for kt in range(S // 64):
        ks = slice(kt * 64, kt * 64 + 64)
        t = _fma32(q @ k[:, :, ks].transpose(-1, -2), SCALE_LOG2, mk[:, None, None, ks])
        mn = torch.maximum(m, t.amax(-1))
        al = torch.exp2(m - mn)
        m = mn
        if mutant != "c_no_l_rescale":
            l = l * al
        if mutant != "b_no_o_rescale":
            o = o * al[..., None]
        e = torch.exp2(t - mn[..., None])
        l = l + e.sum(-1)
        hi = _bf16(e)
        lo = _bf16(e - hi)
        if keep is not None:
            hi, lo = hi * keep[..., ks], lo * keep[..., ks]
        o = o + hi @ v[:, :, ks]
        if mutant != "a_no_lo":
            o = o + lo @ v[:, :, ks]
    ctx = merge_rows((o * (drop_scale(p) / l)[..., None]).to(bf), seq_first)
    lse = m + torch.log2(l)
    return ctx, (lse if mutant == "e_lse_log2" else lse * LN2_32)


def backward_sim(qkv, mask, ctx, dctx, lse, B, S, A, seq_first=False, keep=None, p=0.0, mutant=None):
    """attn_bwd_dkv_kernel + attn_bwd_dq_kernel in fp32: delta = sum dO*O, P = bf16(ex2(fmaf(s, scale*log2e, mask*log2e) - lse*log2e)),
    P~ = P AND keep, dS = bf16(fmaf(P~ * dP, drop_scale*scale, P * -delta*scale)), dV = bf16(drop_scale * P~^T dO), dK = bf16(dS^T Q),
    dQ = bf16(dS K).  Returns dqkv bf16 [T, 3H]."""
    q, k, v = (t.float() for t in split_qkv(qkv, B, S, A, seq_first))
    do = split_rows(dctx, B, S, A, seq_first).float()
    delta = (do * split_rows(ctx, B, S, A, seq_first).float()).sum(-1, keepdim=True)
    mk = torch.zeros(B, S, device=qkv.device) if mask is None else mask.float() * LOG2E32
    t = _fma32(q @ k.transpose(-1, -2), SCALE_LOG2, mk[:, None, None, :]) + (-lse * LOG2E32)[..., None]
    P = _bf16(torch.exp2(t))
    Pt = P * keep if keep is not None else P
    dp = do @ v.transpose(-1, -2)
    dsc = drop_scale(p)
    c1 = float(np.float32(dsc) * np.float32(0.125))
    nd = -delta * 0.125
    dS = _bf16(_fma32(Pt * dp, c1, (Pt if mutant == "f_pdrop_delta" else P) * nd))
    dSk = _bf16(_fma32(Pt * dp, dsc, P * -delta)) if mutant == "g_dk_no_scale" else dS
    grads = (dS @ k, dSk.transpose(-1, -2) @ q, (Pt.transpose(-1, -2) @ do) * dsc)
    return torch.cat([merge_rows(g.to(bf), seq_first) for g in grads], 1)


# ------------------------------------------------------------------------------------------------
# the simulation against the bars
# ------------------------------------------------------------------------------------------------
# (B, S, A, lens, dropout p): an unmasked batch without dropout, and the edge-length batch (with its all-padding row) under dropout
SIM_CASES = {
    "plain": (2, 256, 2, None, 0.0),
    "edges_drop": (len(edge_lens(512)), 512, 1, edge_lens(512), 0.1),
}


@functools.lru_cache(maxsize=None)
def _case(family, case):
    B, S, A, lens, p = SIM_CASES[case]
    seed = 1000 * FAMILIES.index(family) + len(case)
    qkv = family_qkv(family, B, S, A, lens, seed=seed)
    mask = lens_mask(lens, S) if lens is not None else None
    keep = keep_mask(B, S, A, p, seed=seed, stream=3)
    dctx = rand_dctx(B * S, A * HD, seed + 1)
    ref_ctx, ref_lse, ref_dqkv = attention_ref64(qkv, mask, B, S, A, keep=keep, p=p, dctx=dctx)
    return dict(B=B, S=S, A=A, p=p, qkv=qkv, mask=mask, keep=keep, dctx=dctx, ref_ctx=ref_ctx, ref_lse=ref_lse, ref_dqkv=ref_dqkv,
                floor=elem_floor(qkv, mask, B, S, A))


@functools.lru_cache(maxsize=None)
def sim_scores(family, case, mutant=None):
    """bar scores of the simulation (forward and backward) with one mutant or none"""
    c = _case(family, case)
    B, S, A, p = c["B"], c["S"], c["A"], c["p"]
    fwd_mut = mutant if mutant in FWD_MUTANTS else None
    ctx, lse = tiled_forward_sim(c["qkv"], c["mask"], B, S, A, keep=c["keep"], p=p, mutant=fwd_mut)
    sc = forward_scores(ctx, lse, c["ref_ctx"], c["ref_lse"], c["floor"])
    if mutant is None or mutant in BWD_MUTANTS:
        # the backward runs on the correct forward's outputs, as the kernels' backward does
        dqkv = backward_sim(c["qkv"], c["mask"], ctx, c["dctx"], lse, B, S, A, keep=c["keep"], p=p, mutant=mutant)
        yard = backward_yardstick(c["qkv"], c["mask"], ctx, c["dctx"], c["ref_lse"], B, S, A, keep=c["keep"], p=p)
        sc.update(bwd_ratios(dqkv, yard, c["ref_dqkv"], A * HD))
    return sc


@pytest.mark.parametrize("case", sorted(SIM_CASES))
@pytest.mark.parametrize("family", FAMILIES)
def test_correct_simulation_clears_every_bar(family, case):
    sc = sim_scores(family, case)
    assert over_bars(sc) == [], sc


def worst_over_bar(sc):
    return max(v / BARS[k] for k, v in sc.items())


# spike_early: the dominant key sets the row max in the first tile, so its P is exactly 1 and every other P is e^-8 or less of it --
# the lo part of P carries nothing there that survives the bf16 rounding of ctx.  Mutant a is held to the other families.
MUTANT_BLIND = {("a_no_lo", "spike_early")}


@pytest.mark.parametrize("mutant", sorted(FWD_MUTANTS) + sorted(BWD_MUTANTS))
@pytest.mark.parametrize("family", FAMILIES)
def test_mutant_fails_a_bar(family, mutant):
    """Every mutant misses a bar by a clear margin (its score at least 1.5x the bar) on every family, in at least one of the cases:
    b and c need a row max that moves between tiles, d a row whose every key is masked, f dropout."""
    if (mutant, family) in MUTANT_BLIND:
        pytest.skip("the lo part of P is below the bf16 rounding of ctx on this family")
    worst = max(worst_over_bar(sim_scores(family, case, mutant)) for case in SIM_CASES)
    assert worst > 1.5, (family, mutant, worst)


def format_table():
    """per family and case: the correct simulation's bar scores next to each mutant's worst score over its bar"""
    keys = tuple(BARS)
    lines = ["family       case        " + " ".join(f"{k:>9}" for k in keys) + "  | mutant: worst score / bar"]
    for fam in FAMILIES:
        for case in SIM_CASES:
            sc = sim_scores(fam, case)
            muts = [f"{m[0]}={worst_over_bar(sim_scores(fam, case, m)):.3g}" for m in list(FWD_MUTANTS) + list(BWD_MUTANTS)]
            lines.append(f"{fam:<12} {case:<11} " + " ".join(f"{sc[k]:9.3f}" for k in keys) + "  | " + " ".join(muts))
    return "\n".join(lines)


def test_report_table(capsys):
    table = format_table()
    with capsys.disabled():
        print("\nfused attention simulation vs bars (fwd_ratio <= %.2f, elem <= 1, lse <= 1, dq/dk/dv <= %.2f)\n%s"
              % (FWD_RATIO_BAR, BWD_RATIO_BAR, table))
