"""Torch-tensor wrappers over the C ABI (raw pointers + current CUDA stream).

PyTorch is used only for device memory and streams.  Every function requires CUDA tensors and
raises otherwise -- no CPU path exists.
"""
import ctypes

import torch

from . import _lib as L

bf16 = torch.bfloat16
# when a list, gemm() brackets every launch with CUDA events on the launching stream: (e0, e1, flops, tag)
gemm_profile = None


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ptr(t):
    return ctypes.c_void_p(0 if t is None else t.data_ptr())


def _req(t, dtype=None, name="tensor"):
    if not t.is_cuda:
        raise L.DleError(f"{name} must be a CUDA tensor (no CPU fallback in the H100 hot path)")
    if dtype is not None and t.dtype != dtype:
        raise L.DleError(f"{name} must be {dtype}, got {t.dtype}")
    return t


def _row_major_2d(t, name):
    """Accept a 2-D view whose last dim is contiguous; returns leading dimension."""
    if t.dim() != 2 or t.stride(1) != 1:
        raise L.DleError(f"{name} must be 2-D with a contiguous last dim, got shape {tuple(t.shape)} strides {t.stride()}")
    return t.stride(0) if t.size(0) > 1 else max(t.stride(0), t.size(1))


# ------------------------------------------------------------------------------------------------
# GEMM
# ------------------------------------------------------------------------------------------------
def gemm(a, b, *, a_layout=L.LAYOUT_K, b_layout=L.LAYOUT_K, epilogue=L.EPI_BIAS, bias=None, aux=None,
         out=None, out2=None, splits=1, tile_n=0, alpha=1.0, dropout_p=0.0, seed=0, seed_dev=None, dropout_stream=0, colsum_out=None):
    """D[M,N] = alpha * A x B^T with fused epilogue (see include/dle_b200.h).

    a: [M,K] (LAYOUT_K) or [K,M] (LAYOUT_MN);  b: [N,K] (LAYOUT_K) or [K,N] (LAYOUT_MN)."""
    lib = L.load()
    _req(a, bf16, "A"); _req(b, bf16, "B")
    lda, ldb = _row_major_2d(a, "A"), _row_major_2d(b, "B")
    M, K = (a.shape if a_layout == L.LAYOUT_K else (a.shape[1], a.shape[0]))
    N, Kb = (b.shape if b_layout == L.LAYOUT_K else (b.shape[1], b.shape[0]))
    if K != Kb:
        raise L.DleError(f"GEMM reduction dims differ: {K} vs {Kb}")
    f32_out = epilogue in (L.EPI_ATOMIC_F32, L.EPI_F32)
    if out is None:
        out = (torch.zeros if epilogue == L.EPI_ATOMIC_F32 else torch.empty)(
            (M, N), device=a.device, dtype=torch.float32 if f32_out else bf16)
    _req(out, torch.float32 if f32_out else bf16, "out")
    if epilogue == L.EPI_BIAS_GELU and out2 is None:
        out2 = torch.empty((M, N), device=a.device, dtype=bf16)
    args = L.GemmArgs()
    args.A, args.B, args.out = a.data_ptr(), b.data_ptr(), out.data_ptr()
    args.out2 = 0 if out2 is None else _req(out2, bf16, "out2").data_ptr()
    args.bias = 0 if bias is None else _req(bias, bf16, "bias").data_ptr()
    args.aux = 0 if aux is None else _req(aux, bf16, "aux").data_ptr()
    args.M, args.N, args.K = M, N, K
    args.a_layout, args.b_layout = a_layout, b_layout
    args.lda, args.ldb = lda, ldb
    args.ldo = _row_major_2d(out, "out")
    args.ldo2 = 0 if out2 is None else _row_major_2d(out2, "out2")
    args.ld_aux = 0 if aux is None else _row_major_2d(aux, "aux")
    args.epilogue, args.splits, args.tile_n = epilogue, splits, tile_n
    args.alpha, args.dropout_p = alpha, dropout_p
    args.dropout_stream, args.seed = dropout_stream, seed
    args.seed_dev = 0 if seed_dev is None else seed_dev.data_ptr()
    args.colsum_out = 0 if colsum_out is None else _req(colsum_out, torch.float32, "colsum_out").data_ptr()
    if gemm_profile is not None:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
    L.launch_count["n"] += 1; L.check(lib.dle_gemm_bf16(ctypes.byref(args), _stream()), "dle_gemm_bf16")
    if gemm_profile is not None:
        e1.record()
        gemm_profile.append((e0, e1, 2.0 * M * N * K, (M, N, K, a_layout, b_layout, epilogue)))
    return (out, out2) if epilogue == L.EPI_BIAS_GELU else out


# ------------------------------------------------------------------------------------------------
# attention
# ------------------------------------------------------------------------------------------------
def attn_fwd(qkv, mask, B, S, A, dropout_p=0.0, seed=0, dropout_stream=0, seq_first=False, seed_dev=None):
    lib = L.load()
    _req(qkv, bf16, "qkv")
    ctx = torch.empty((B * S, A * 64), device=qkv.device, dtype=bf16)
    lse = torch.empty((B, A, S), device=qkv.device, dtype=torch.float32)
    if mask is not None:
        _req(mask, torch.float32, "mask")
    L.launch_count["n"] += 1; L.check(lib.dle_attn_fwd(_ptr(qkv), _ptr(mask), _ptr(ctx), _ptr(lse), B, S, A, 1 if seq_first else 0, dropout_p, seed,
                             _ptr(seed_dev), dropout_stream, _stream()), "dle_attn_fwd")
    return ctx, lse


def attn_bwd(qkv, mask, ctx, dctx, lse, B, S, A, dropout_p=0.0, seed=0, dropout_stream=0, seq_first=False, dbias=None, seed_dev=None):
    """dbias: optional zeroed fp32 [3H] receiving the column sums of dqkv (q/k/v bias gradients)."""
    lib = L.load()
    dqkv = torch.empty_like(qkv)
    delta = torch.empty((B, A, S), device=qkv.device, dtype=torch.float32)
    L.launch_count["n"] += 2; L.check(lib.dle_attn_bwd(_ptr(qkv), _ptr(mask), _ptr(ctx), _ptr(_req(dctx, bf16, "dctx")), _ptr(lse), _ptr(dqkv),
                             _ptr(delta), _ptr(dbias), B, S, A, 1 if seq_first else 0, dropout_p, seed, _ptr(seed_dev), dropout_stream, _stream()), "dle_attn_bwd")
    return dqkv


# ------------------------------------------------------------------------------------------------
# LayerNorm family
# ------------------------------------------------------------------------------------------------
def add_ln_fwd(x, gamma, beta, *, bias=None, residual=None, eps=1e-12, dropout_p=0.0, seed=0, dropout_stream=0,
               save_z=True, seed_dev=None):
    lib = L.load()
    _req(x, bf16, "x")
    T, H = x.shape
    fused = bias is not None or residual is not None or dropout_p > 0.0
    z = torch.empty_like(x) if fused else None
    y = torch.empty_like(x)
    mean = torch.empty(T, device=x.device, dtype=torch.float32)
    rstd = torch.empty(T, device=x.device, dtype=torch.float32)
    L.launch_count["n"] += 1; L.check(lib.dle_add_ln_fwd(_ptr(x), _ptr(bias), _ptr(residual), _ptr(gamma), _ptr(beta), _ptr(z), _ptr(y), _ptr(mean),
                               _ptr(rstd), T, H, eps, dropout_p, seed, _ptr(seed_dev), dropout_stream, _stream()), "dle_add_ln_fwd")
    return y, (z if z is not None else x), mean, rstd


def add_ln_bwd(dy, z, mean, rstd, gamma, *, dropout_p=0.0, seed=0, dropout_stream=0, want_dbias=True, out_dtype=torch.float32, seed_dev=None):
    """returns dz, dx (== dz when no dropout), dgamma, dbeta, dbias ([H] each, fp32 or bf16 per out_dtype)."""
    lib = L.load()
    T, H = dy.shape
    n_part = lib.dle_ln_bwd_partials_h(T, H)
    parts = torch.empty((3, n_part, H), device=dy.device, dtype=torch.float32)
    dz = torch.empty_like(dy)
    dx = torch.empty_like(dy) if dropout_p > 0.0 else None
    L.launch_count["n"] += 1; L.check(lib.dle_add_ln_bwd(_ptr(dy), _ptr(z), _ptr(mean), _ptr(rstd), _ptr(gamma), _ptr(dz), _ptr(dx), _ptr(parts[0]),
                               _ptr(parts[1]), _ptr(parts[2]) if want_dbias else None, T, H, dropout_p, seed,
                               _ptr(seed_dev), dropout_stream, _stream()), "dle_add_ln_bwd")
    na = 3 if want_dbias else 2
    red = torch.empty((na, H), device=dy.device, dtype=out_dtype)
    L.launch_count["n"] += 1; L.check(lib.dle_colsum_finalize_batched(_ptr(parts), na, n_part, H, _ptr(red), L.DLE_DTYPE_F32 if out_dtype == torch.float32 else L.DLE_DTYPE_BF16, 0, _stream()),
                                      "dle_colsum_finalize_batched")
    return (dz, dx if dx is not None else dz, *red.unbind(0))


def colsum(x):
    """fp32 column sums of a bf16 [T,N] matrix (bias gradients)."""
    lib = L.load()
    _req(x, bf16, "x")
    T, N = x.shape
    n_part = lib.dle_colsum_partials(T)
    part = torch.empty((n_part, N), device=x.device, dtype=torch.float32)
    L.launch_count["n"] += 1; L.check(lib.dle_colsum_bf16(_ptr(x), T, N, _row_major_2d(x, "x"), _ptr(part), _stream()), "dle_colsum_bf16")
    out = torch.empty(N, device=x.device, dtype=torch.float32)
    L.launch_count["n"] += 1; L.check(lib.dle_colsum_finalize(_ptr(part), n_part, N, _ptr(out), L.DLE_DTYPE_F32, 0, _stream()), "dle_colsum_finalize")
    return out


def bias_gelu_fwd(x, bias=None, save_u=True):
    lib = L.load()
    _req(x, bf16, "x")
    T, N = x.shape
    u = torch.empty_like(x) if (save_u and bias is not None) else None
    y = torch.empty_like(x)
    L.launch_count["n"] += 1; L.check(lib.dle_bias_gelu_fwd(_ptr(x), _ptr(bias), _ptr(u), _ptr(y), T, N, _stream()), "dle_bias_gelu_fwd")
    return y, (u if u is not None else x)


def bias_gelu_bwd(dy, u):
    lib = L.load()
    T, N = dy.shape
    du = torch.empty_like(dy)
    L.launch_count["n"] += 1; L.check(lib.dle_bias_gelu_bwd(_ptr(dy), _ptr(u), _ptr(du), T, N, _stream()), "dle_bias_gelu_bwd")
    return du


# ------------------------------------------------------------------------------------------------
# embeddings / gathers / casts
# ------------------------------------------------------------------------------------------------
def embed_ln_fwd(input_ids, token_type_ids, word, pos, typ, gamma, beta, *, eps=1e-12, dropout_p=0.0, seed=0,
                 dropout_stream=0, err_flag=None, seed_dev=None):
    lib = L.load()
    _req(input_ids, torch.int64, "input_ids"); _req(token_type_ids, torch.int64, "token_type_ids"); _req(word, bf16, "word")
    B, S = input_ids.shape
    H = word.shape[1]
    T = B * S
    z = torch.empty((T, H), device=word.device, dtype=bf16)
    y = torch.empty((T, H), device=word.device, dtype=bf16)
    mean = torch.empty(T, device=word.device, dtype=torch.float32)
    rstd = torch.empty(T, device=word.device, dtype=torch.float32)
    L.launch_count["n"] += 1; L.check(lib.dle_embed_ln_fwd(_ptr(input_ids), _ptr(token_type_ids), _ptr(word), _ptr(pos), _ptr(typ), _ptr(gamma), _ptr(beta),
                                 _ptr(z), _ptr(y), _ptr(mean), _ptr(rstd), B, S, H, word.shape[0], pos.shape[0], typ.shape[0],
                                 eps, dropout_p, seed, _ptr(seed_dev), dropout_stream, _ptr(err_flag), _stream()), "dle_embed_ln_fwd")
    return y, z, mean, rstd


def embed_ln_bwd(dy, z, mean, rstd, gamma, input_ids, token_type_ids, V, P, NT, *, dropout_p=0.0, seed=0, dropout_stream=0, seed_dev=None):
    """returns fp32 dword [V,H], dpos [P,H], dtype [NT,H], dgamma [H], dbeta [H]."""
    lib = L.load()
    B, S = input_ids.shape
    T, H = dy.shape
    dword = torch.zeros((V, H), device=dy.device, dtype=torch.float32)
    dpos = torch.zeros((P, H), device=dy.device, dtype=torch.float32)
    dtyp = torch.zeros((NT, H), device=dy.device, dtype=torch.float32)
    n_part = lib.dle_ln_bwd_partials(T)
    parts = torch.empty((2, n_part, H), device=dy.device, dtype=torch.float32)
    L.launch_count["n"] += 1; L.check(lib.dle_embed_ln_bwd(_ptr(dy), _ptr(z), _ptr(mean), _ptr(rstd), _ptr(gamma), _ptr(input_ids), _ptr(token_type_ids),
                                 _ptr(dword), _ptr(dpos), _ptr(dtyp), _ptr(parts[0]), _ptr(parts[1]), B, S, H, dropout_p, seed,
                                 _ptr(seed_dev), dropout_stream, _stream()), "dle_embed_ln_bwd")
    red = torch.empty((2, H), device=dy.device, dtype=torch.float32)
    L.launch_count["n"] += 1; L.check(lib.dle_colsum_finalize_batched(_ptr(parts), 2, n_part, H, _ptr(red), L.DLE_DTYPE_F32, 0, _stream()),
                                      "dle_colsum_finalize_batched")
    return dword, dpos, dtyp, red[0], red[1]


def gather_rows(x, idx, err_flag=None):
    lib = L.load()
    _req(x, bf16, "x"); _req(idx, torch.int64, "idx")
    out = torch.empty((idx.numel(), x.shape[1]), device=x.device, dtype=bf16)
    if idx.numel() == 0:
        return out
    L.launch_count["n"] += 1; L.check(lib.dle_gather_rows(_ptr(x), _ptr(idx), _ptr(out), idx.numel(), x.shape[1], x.shape[0], _ptr(err_flag), _stream()),
            "dle_gather_rows")
    return out


def scatter_rows(dy, idx, n_rows):
    lib = L.load()
    dx = torch.zeros((n_rows, dy.shape[1]), device=dy.device, dtype=bf16)
    if idx.numel() == 0:
        return dx
    L.launch_count["n"] += 1; L.check(lib.dle_scatter_rows(_ptr(dy), _ptr(idx), _ptr(dx), idx.numel(), dy.shape[1], n_rows, _stream()), "dle_scatter_rows")
    return dx


def softmax_ce_fwd(logits, labels, ignore_index=-1, err_flag=None):
    """fp32 log-sum-exp and per-row loss of bf16 logits [rows, V]; returns (lse [rows], loss_rows [rows]) fp32."""
    lib = L.load()
    _req(logits, bf16, "logits"); _req(labels, torch.int64, "labels")
    rows, V = logits.shape
    ld = _row_major_2d(logits, "logits")
    lse = torch.empty(rows, device=logits.device, dtype=torch.float32)
    loss = torch.empty(rows, device=logits.device, dtype=torch.float32)
    L.launch_count["n"] += 1; L.check(lib.dle_softmax_ce_fwd(_ptr(logits), _ptr(labels), _ptr(lse), _ptr(loss), rows, V, ld, ignore_index, _ptr(err_flag), _stream()),
                                      "dle_softmax_ce_fwd")
    return lse, loss


def softmax_ce_bwd(logits, labels, lse, grad_scale, ignore_index=-1):
    """dlogits (bf16, same shape) = (softmax - onehot) * grad_scale for counted rows; grad_scale: fp32 device scalar."""
    lib = L.load()
    rows, V = logits.shape
    out = torch.empty((rows, V), device=logits.device, dtype=bf16)
    L.launch_count["n"] += 1; L.check(lib.dle_softmax_ce_bwd(_ptr(logits), _ptr(labels), _ptr(lse), _ptr(_req(grad_scale, torch.float32, "grad_scale")), _ptr(out), rows, V,
                                                            _row_major_2d(logits, "logits"), V, ignore_index, _stream()), "dle_softmax_ce_bwd")
    return out


def advance_u64(counter, delta=1):
    """counter (int64/uint64 device tensor, 1 element) += delta on the current stream; graph-capturable."""
    lib = L.load()
    _req(counter, None, "counter")
    L.launch_count["n"] += 1; L.check(lib.dle_advance_u64(_ptr(counter), int(delta), _stream()), "dle_advance_u64")


def cast_f32_to_bf16(x, out=None):
    lib = L.load()
    _req(x, torch.float32, "x")
    out = torch.empty(x.shape, device=x.device, dtype=bf16) if out is None else out
    L.launch_count["n"] += 1; L.check(lib.dle_cast_f32_to_bf16(_ptr(x), _ptr(out), x.numel(), _stream()), "dle_cast_f32_to_bf16")
    return out


def cast_bf16_to_f32(x, out=None):
    lib = L.load()
    _req(x, bf16, "x")
    out = torch.empty(x.shape, device=x.device, dtype=torch.float32) if out is None else out
    L.launch_count["n"] += 1; L.check(lib.dle_cast_bf16_to_f32(_ptr(x), _ptr(out), x.numel(), _stream()), "dle_cast_bf16_to_f32")
    return out
