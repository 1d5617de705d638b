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

    a: [M,K] (LAYOUT_K) or [K,M] (LAYOUT_MN);  b: [N,K] (LAYOUT_K) or [K,N] (LAYOUT_MN).
    EPI_BIAS_GELU returns (out, out2 = pre-activation u); out2=False skips the store of u (inference) and returns (out, None)."""
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
    if out2 is False:
        if epilogue != L.EPI_BIAS_GELU:
            raise L.DleError("out2=False applies to EPI_BIAS_GELU only")
        out2 = None
    elif epilogue == L.EPI_BIAS_GELU and out2 is None:
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


def attn_fwd_varlen(qkv, cu_seqlens, B, max_seqlen, A, out=None):
    """Inference attention over packed sequences: qkv [T, 3*A*64] bf16, cu_seqlens int32 [B+1] on the device (sequence b is rows
    cu_seqlens[b] .. cu_seqlens[b+1], each at most max_seqlen <= 512 long).  Returns ctx [T, A*64] (written into `out` when given;
    rows outside every sequence are left as they are); no mask, dropout or lse."""
    lib = L.load()
    _req(qkv, bf16, "qkv"); _req(cu_seqlens, torch.int32, "cu_seqlens")
    if qkv.dim() != 2 or qkv.shape[1] != 3 * A * 64 or not qkv.is_contiguous():
        raise L.DleError(f"qkv must be a contiguous [T, {3 * A * 64}] tensor, got shape {tuple(qkv.shape)}")
    if cu_seqlens.shape != (B + 1,) or not cu_seqlens.is_contiguous():
        raise L.DleError(f"cu_seqlens must be a contiguous [{B + 1}] tensor, got shape {tuple(cu_seqlens.shape)}")
    ctx = torch.empty((qkv.shape[0], A * 64), device=qkv.device, dtype=bf16) if out is None else out
    if ctx.shape != (qkv.shape[0], A * 64) or not ctx.is_contiguous():
        raise L.DleError(f"out must be a contiguous [{qkv.shape[0]}, {A * 64}] tensor")
    _req(ctx, bf16, "out")
    if qkv.shape[0] == 0:
        return ctx
    L.launch_count["n"] += 1; L.check(lib.dle_attn_fwd_varlen(_ptr(qkv), _ptr(cu_seqlens), _ptr(ctx), B, max_seqlen, A, _stream()),
                                      "dle_attn_fwd_varlen")
    return ctx


def _check_varlen(qkv, cu_seqlens, B, A):
    _req(qkv, bf16, "qkv"); _req(cu_seqlens, torch.int32, "cu_seqlens")
    if qkv.dim() != 2 or qkv.shape[1] != 3 * A * 64 or not qkv.is_contiguous():
        raise L.DleError(f"qkv must be a contiguous [T, {3 * A * 64}] tensor, got shape {tuple(qkv.shape)}")
    if cu_seqlens.shape != (B + 1,) or not cu_seqlens.is_contiguous():
        raise L.DleError(f"cu_seqlens must be a contiguous [{B + 1}] tensor, got shape {tuple(cu_seqlens.shape)}")


def _check_rows(t, rows, cols, dtype, name):
    _req(t, dtype, name)
    if tuple(t.shape) != (rows, cols) or not t.is_contiguous():
        raise L.DleError(f"{name} must be a contiguous [{rows}, {cols}] tensor, got shape {tuple(t.shape)}")


def attn_fwd_varlen_train(qkv, cu_seqlens, B, max_seqlen, A, drop_stride, dropout_p=0.0, seed=0, dropout_stream=0, seed_dev=None):
    """Training attention over packed sequences (the arguments of attn_fwd_varlen, plus attn_fwd's dropout).  Returns ctx [T, A*64]
    and lse fp32 [A, T]; rows outside every sequence are left as they are.  The keep bits of (sequence b, head h, query q, key k) are
    keyed at ((b*A + h)*drop_stride + q)*drop_stride + k: drop_stride = S (a multiple of 64, max_seqlen <= drop_stride <= 512) draws
    attn_fwd's bits for a right-padded batch of length S."""
    lib = L.load()
    _check_varlen(qkv, cu_seqlens, B, A)
    T = qkv.shape[0]
    ctx = torch.empty((T, A * 64), device=qkv.device, dtype=bf16)
    lse = torch.empty((A, T), device=qkv.device, dtype=torch.float32)
    if T == 0:
        return ctx, lse
    L.launch_count["n"] += 1; L.check(lib.dle_attn_fwd_varlen_train(_ptr(qkv), _ptr(cu_seqlens), _ptr(ctx), _ptr(lse), T, B, max_seqlen, A,
                                                                    drop_stride, dropout_p, seed, _ptr(seed_dev), dropout_stream, _stream()),
                                      "dle_attn_fwd_varlen_train")
    return ctx, lse


def attn_bwd_varlen(qkv, cu_seqlens, ctx, dctx, lse, B, max_seqlen, A, drop_stride, dropout_p=0.0, seed=0, dropout_stream=0, dbias=None,
                    seed_dev=None, out=None):
    """Backward of attn_fwd_varlen_train: dqkv [T, 3*A*64] (written into `out` when given; rows outside every sequence are left as
    they are).  dbias: optional zeroed fp32 [3*A*64] receiving the column sums of dqkv's rows inside the sequences."""
    lib = L.load()
    _check_varlen(qkv, cu_seqlens, B, A)
    T, H = qkv.shape[0], A * 64
    _check_rows(ctx, T, H, bf16, "ctx"); _check_rows(dctx, T, H, bf16, "dctx"); _check_rows(lse, A, T, torch.float32, "lse")
    dqkv = torch.empty_like(qkv) if out is None else out
    _check_rows(dqkv, T, 3 * H, bf16, "out")
    if dbias is not None and (tuple(dbias.shape) != (3 * H,) or not _req(dbias, torch.float32, "dbias").is_contiguous()):
        raise L.DleError(f"dbias must be a contiguous fp32 [{3 * H}] tensor")
    if T == 0:
        return dqkv
    delta = torch.empty((A, T), device=qkv.device, dtype=torch.float32)
    L.launch_count["n"] += 3; L.check(lib.dle_attn_bwd_varlen(_ptr(qkv), _ptr(cu_seqlens), _ptr(ctx), _ptr(dctx), _ptr(lse), _ptr(dqkv),
                                                              _ptr(delta), _ptr(dbias), T, B, max_seqlen, A, drop_stride, dropout_p, seed,
                                                              _ptr(seed_dev), dropout_stream, _stream()), "dle_attn_bwd_varlen")
    return dqkv


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
def _check_positions(position_ids, B, S):
    if position_ids is not None:
        _req(position_ids, torch.int64, "position_ids")
        if tuple(position_ids.shape) != (B, S) or not position_ids.is_contiguous():
            raise L.DleError(f"position_ids must be a contiguous [{B}, {S}] tensor, got shape {tuple(position_ids.shape)}")
    return position_ids


def embed_ln_fwd(input_ids, token_type_ids, word, pos, typ, gamma, beta, *, eps=1e-12, dropout_p=0.0, seed=0,
                 dropout_stream=0, err_flag=None, seed_dev=None, position_ids=None):
    """position_ids: optional int64 [B, S] (None = arange(S) in every row); a position outside the table sets err_flag."""
    lib = L.load()
    _req(input_ids, torch.int64, "input_ids"); _req(token_type_ids, torch.int64, "token_type_ids"); _req(word, bf16, "word")
    B, S = input_ids.shape
    _check_positions(position_ids, B, S)
    H = word.shape[1]
    T = B * S
    z = torch.empty((T, H), device=word.device, dtype=bf16)
    y = torch.empty((T, H), device=word.device, dtype=bf16)
    mean = torch.empty(T, device=word.device, dtype=torch.float32)
    rstd = torch.empty(T, device=word.device, dtype=torch.float32)
    L.launch_count["n"] += 1; L.check(lib.dle_embed_ln_fwd(_ptr(input_ids), _ptr(token_type_ids), _ptr(word), _ptr(pos), _ptr(typ), _ptr(gamma), _ptr(beta),
                                 _ptr(z), _ptr(y), _ptr(mean), _ptr(rstd), B, S, H, word.shape[0], pos.shape[0], typ.shape[0],
                                 eps, dropout_p, seed, _ptr(seed_dev), dropout_stream, _ptr(err_flag), _stream(), _ptr(position_ids)), "dle_embed_ln_fwd")
    return y, z, mean, rstd


def embed_ln_bwd(dy, z, mean, rstd, gamma, input_ids, token_type_ids, V, P, NT, *, dropout_p=0.0, seed=0, dropout_stream=0, seed_dev=None,
                 position_ids=None):
    """returns fp32 dword [V,H], dpos [P,H], dtype [NT,H], dgamma [H], dbeta [H].  position_ids: those the forward was given."""
    lib = L.load()
    B, S = input_ids.shape
    _check_positions(position_ids, B, S)
    T, H = dy.shape
    dword = torch.zeros((V, H), device=dy.device, dtype=torch.float32)
    dpos = torch.zeros((P, H), device=dy.device, dtype=torch.float32)
    dtyp = torch.zeros((NT, H), device=dy.device, dtype=torch.float32)
    n_part = lib.dle_ln_bwd_partials(T)
    parts = torch.empty((2, n_part, H), device=dy.device, dtype=torch.float32)
    L.launch_count["n"] += 1; L.check(lib.dle_embed_ln_bwd(_ptr(dy), _ptr(z), _ptr(mean), _ptr(rstd), _ptr(gamma), _ptr(input_ids), _ptr(token_type_ids),
                                 _ptr(dword), _ptr(dpos), _ptr(dtyp), _ptr(parts[0]), _ptr(parts[1]), B, S, H, dropout_p, seed,
                                 _ptr(seed_dev), dropout_stream, _stream(), _ptr(position_ids)), "dle_embed_ln_bwd")
    red = torch.empty((2, H), device=dy.device, dtype=torch.float32)
    L.launch_count["n"] += 1; L.check(lib.dle_colsum_finalize_batched(_ptr(parts), 2, n_part, H, _ptr(red), L.DLE_DTYPE_F32, 0, _stream()),
                                      "dle_colsum_finalize_batched")
    return dword, dpos, dtyp, red[0], red[1]


def segment_table(mask, k, err_flag=None):
    """Segment table of a packed batch (include/dle_b200.h, dle_segment_table): mask int64 [B, S] holds each token's sample number
    (1..k, contiguous and increasing, 0 on the padding tail).  Returns cu_seqlens int32 [B*(k+1) + 1], position_ids int64 [B, S] and
    cls_index int64 [B*k]; a malformed row sets err_flag and becomes one tail segment."""
    lib = L.load()
    _req(mask, torch.int64, "mask")
    if mask.dim() != 2 or not mask.is_contiguous():
        raise L.DleError(f"mask must be a contiguous [B, S] tensor, got shape {tuple(mask.shape)}")
    B, S = mask.shape
    cu = torch.empty(B * (k + 1) + 1, device=mask.device, dtype=torch.int32)
    pos = torch.empty((B, S), device=mask.device, dtype=torch.int64)
    cls = torch.empty(B * k, device=mask.device, dtype=torch.int64)
    L.launch_count["n"] += 1; L.check(lib.dle_segment_table(_ptr(mask), B, S, k, _ptr(cu), _ptr(pos), _ptr(cls), _ptr(err_flag), _stream()),
                                      "dle_segment_table")
    return cu, pos, cls


_DTYPE_CODE = {torch.float32: L.DLE_DTYPE_F32, bf16: L.DLE_DTYPE_BF16}


def _span_dtype(t, name):
    _req(t, name=name)
    if t.dtype not in _DTYPE_CODE:
        raise L.DleError(f"{name} must be bfloat16 or float32, got {t.dtype}")
    return _DTYPE_CODE[t.dtype]


def span_logits_unpack(logits, cu_seqlens, B, S, k, fill=-10000.0):
    """Per-sample span logits of a packed batch (include/dle_b200.h, dle_span_logits_unpack): logits [B*S, 2] (bf16 or fp32, last dim
    contiguous) and cu_seqlens of segment_table(mask, k) -> (start, end), each [B*k, S] of the logits' dtype, left-aligned per sample
    and `fill` everywhere else."""
    lib = L.load()
    code = _span_dtype(logits, "logits")
    _req(cu_seqlens, torch.int32, "cu_seqlens")
    if tuple(logits.shape) != (B * S, 2) or cu_seqlens.numel() != B * (k + 1) + 1 or not cu_seqlens.is_contiguous():
        raise L.DleError(f"span_logits_unpack: logits must be [{B * S}, 2] and cu_seqlens [{B * (k + 1) + 1}], got "
                         f"{tuple(logits.shape)} and {tuple(cu_seqlens.shape)}")
    ld = _row_major_2d(logits, "logits")
    start = torch.empty((B * k, S), device=logits.device, dtype=logits.dtype)
    end = torch.empty_like(start)
    L.launch_count["n"] += 1; L.check(lib.dle_span_logits_unpack(_ptr(logits), ld, _ptr(cu_seqlens), B, S, k, code, fill, _ptr(start), _ptr(end),
                                                                 _stream()), "dle_span_logits_unpack")
    return start, end


def span_logits_pack_grad(dstart, dend, cu_seqlens, B, S, k):
    """The gradient of span_logits_unpack: dstart, dend [B*k, S] -> dlogits [B*S, 2] of their dtype (0 at every tail token)."""
    lib = L.load()
    code = _span_dtype(dstart, "dstart")
    _req(dend, dstart.dtype, "dend"); _req(cu_seqlens, torch.int32, "cu_seqlens")
    for t, name in ((dstart, "dstart"), (dend, "dend")):
        if tuple(t.shape) != (B * k, S) or not t.is_contiguous():
            raise L.DleError(f"{name} must be a contiguous [{B * k}, {S}] tensor, got shape {tuple(t.shape)}")
    if cu_seqlens.numel() != B * (k + 1) + 1 or not cu_seqlens.is_contiguous():
        raise L.DleError(f"cu_seqlens must hold {B * (k + 1) + 1} entries, got {tuple(cu_seqlens.shape)}")
    dlogits = torch.empty((B * S, 2), device=dstart.device, dtype=dstart.dtype)
    L.launch_count["n"] += 1; L.check(lib.dle_span_logits_pack_grad(_ptr(dstart), _ptr(dend), _ptr(cu_seqlens), B, S, k, code, _ptr(dlogits), 2,
                                                                    _stream()), "dle_span_logits_pack_grad")
    return dlogits


def _cls_head_x(x, w):
    """x as the head kernels take it (bf16 [R, H], row stride a multiple of 8, 16-byte aligned) and its row stride."""
    _req(x, bf16, "x"); _req(w, bf16, "w")
    if x.dim() != 2 or w.dim() != 2 or x.shape[1] != w.shape[1] or not w.is_contiguous():
        raise L.DleError(f"cls_head: x must be [R, H] and w a contiguous [L, H], got {tuple(x.shape)} and {tuple(w.shape)}")
    ld = _row_major_2d(x, "x")
    if ld % 8 or x.data_ptr() % 16:
        x = x.contiguous()
        ld = x.shape[1]
    return x, ld


def cls_head_fwd(x, w, b, dropout_p=0.0, seed=0, dropout_stream=0, seed_dev=None):
    """Sequence-classification head (include/dle_b200.h, dle_cls_head_fwd): x [R, H] bf16, w [L, H] bf16, b [L] bf16 or fp32 ->
    logits [R, L] of b's dtype, logits = dropout(x) @ w^T + b with the hidden-dropout keep bits of element r*H + c."""
    lib = L.load()
    x, ldx = _cls_head_x(x, w)
    code = _span_dtype(b, "b")
    R, H = x.shape
    n_lab = w.shape[0]
    if tuple(b.shape) != (n_lab,) or not b.is_contiguous():
        raise L.DleError(f"b must be a contiguous [{n_lab}] tensor, got shape {tuple(b.shape)}")
    logits = torch.empty((R, n_lab), device=x.device, dtype=b.dtype)
    L.launch_count["n"] += 1; L.check(lib.dle_cls_head_fwd(_ptr(x), ldx, _ptr(w), _ptr(b), R, H, n_lab, code, dropout_p, seed, _ptr(seed_dev),
                                                           dropout_stream, _ptr(logits), _stream()), "dle_cls_head_fwd")
    return logits


def cls_head_bwd(dlogits, x, w, dropout_p=0.0, seed=0, dropout_stream=0, seed_dev=None):
    """The gradients of cls_head_fwd for dlogits [R, L] (bf16 or fp32, the parameter dtype): (dx [R, H] bf16, dw [L, H], db [L]), dw and
    db of dlogits' dtype, summed over rows in a fixed order.  The dropout arguments must be those of the forward."""
    lib = L.load()
    x, ldx = _cls_head_x(x, w)
    code = _span_dtype(dlogits, "dlogits")
    R, H = x.shape
    n_lab = w.shape[0]
    if tuple(dlogits.shape) != (R, n_lab) or not dlogits.is_contiguous():
        raise L.DleError(f"dlogits must be a contiguous [{R}, {n_lab}] tensor, got shape {tuple(dlogits.shape)}")
    n_part = lib.dle_cls_head_bwd_partials(R)
    if n_part <= 0:
        raise L.DleError(f"cls_head_bwd: R = {R} rows")
    part = torch.empty(n_part * n_lab * (H + 1), device=x.device, dtype=torch.float32)
    dx = torch.empty((R, H), device=x.device, dtype=bf16)
    dw = torch.empty((n_lab, H), device=x.device, dtype=dlogits.dtype)
    db = torch.empty((n_lab,), device=x.device, dtype=dlogits.dtype)
    L.launch_count["n"] += 3; L.check(lib.dle_cls_head_bwd(_ptr(dlogits), _ptr(x), ldx, _ptr(w), R, H, n_lab, code, dropout_p, seed,
                                                           _ptr(seed_dev), dropout_stream, _ptr(dx), _ptr(part), _ptr(dw), _ptr(db),
                                                           _stream()), "dle_cls_head_bwd")
    return dx, dw, db


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


# ------------------------------------------------------------------------------------------------
# distillation losses (csrc/distill_sm90.cu)
# ------------------------------------------------------------------------------------------------
def _head_block(t, A, name):
    """A 2-D bf16 view whose first 64*A columns are the heads' blocks (last dim contiguous); returns its row stride."""
    _req(t, bf16, name)
    ld = _row_major_2d(t, name)
    if t.shape[1] < 64 * A:
        raise L.DleError(f"{name} has {t.shape[1]} columns, fewer than 64 * A = {64 * A}")
    return ld


def relkl_fwd(xs, ys, xt, yt, mask_s, mask_t, B, S, A, scale_s, scale_t, where_rule, seq_first, norm):
    """loss = norm * sum over rows of KL(softmax(t) || softmax(s)); s / t = scale * X Y^T (+ mask) per (b, h) (see dle_relkl_fwd).
    xs, ys, xt, yt: 2-D bf16 views starting at head 0's column block; masks fp32 [B, S] or None.  Returns (loss [] fp32, lse_s,
    lse_t [B, A, S])."""
    lib = L.load()
    ld_s, ld_t = _head_block(xs, A, "xs"), _head_block(xt, A, "xt")
    if _head_block(ys, A, "ys") != ld_s or _head_block(yt, A, "yt") != ld_t:
        raise L.DleError("X and Y of one model must share a row stride")
    for m, n in ((mask_s, "mask_s"), (mask_t, "mask_t")):
        if m is not None:
            _req(m, torch.float32, n)
    dev = xs.device
    lse_s = torch.empty((B, A, S), device=dev, dtype=torch.float32)
    lse_t = torch.empty((B, A, S), device=dev, dtype=torch.float32)
    n_part = lib.dle_relkl_partials(B, S, A)
    L.check(n_part if n_part < 0 else 0, "dle_relkl_partials")
    ws = torch.empty(n_part + 1, device=dev, dtype=torch.float32)
    L.launch_count["n"] += 2; L.check(lib.dle_relkl_fwd(_ptr(xs), _ptr(ys), _ptr(xt), _ptr(yt), ld_s, ld_t, _ptr(mask_s), _ptr(mask_t),
                                                        scale_s, scale_t, 1 if where_rule else 0, B, S, A, 1 if seq_first else 0, norm,
                                                        _ptr(lse_s), _ptr(lse_t), _ptr(ws[1:]), _ptr(ws), _stream()), "dle_relkl_fwd")
    return ws[0], lse_s, lse_t


def relkl_bwd(xs, ys, xt, yt, mask_s, mask_t, B, S, A, scale_s, scale_t, where_rule, seq_first, lse_s, lse_t, grad_scale, norm, dx, dy,
              dzero=None):
    """Gradient of relkl_fwd's loss times grad_scale (fp32 device scalar) into the bf16 views dx (= dS Y_s) and dy (= dS^T X_s); when
    dx and dy are the same view (X = Y) the two terms are summed.  dzero: a view zero-filled per head block, or None."""
    lib = L.load()
    ld_s, ld_t = _head_block(xs, A, "xs"), _head_block(xt, A, "xt")
    ld_d = _head_block(dx, A, "dx")
    if _head_block(dy, A, "dy") != ld_d or (dzero is not None and _head_block(dzero, A, "dzero") != ld_d):
        raise L.DleError("dx, dy and dzero must share a row stride")
    L.launch_count["n"] += 2; L.check(lib.dle_relkl_bwd(_ptr(xs), _ptr(ys), _ptr(xt), _ptr(yt), ld_s, ld_t, _ptr(mask_s), _ptr(mask_t),
                                                        scale_s, scale_t, 1 if where_rule else 0, B, S, A, 1 if seq_first else 0,
                                                        _ptr(lse_s), _ptr(lse_t), _ptr(_req(grad_scale, torch.float32, "grad_scale")),
                                                        norm, _ptr(dx), _ptr(dy), _ptr(dzero), ld_d, _stream()), "dle_relkl_bwd")


def cosine_rows_fwd(x, y):
    """mean over rows of 1 - cos(x_r, y_r) (torch's CosineEmbeddingLoss with target 1) on bf16 [rows, H]; returns a [] fp32 tensor."""
    lib = L.load()
    _req(x, bf16, "x"); _req(y, bf16, "y")
    if x.shape != y.shape or x.dim() != 2:
        raise L.DleError(f"cosine rows need two [rows, H] tensors of one shape, got {tuple(x.shape)} and {tuple(y.shape)}")
    rows, H = x.shape
    n_part = lib.dle_cosine_rows_partials(rows)
    L.check(n_part if n_part < 0 else 0, "dle_cosine_rows_partials")
    ws = torch.empty(n_part + 1, device=x.device, dtype=torch.float32)
    L.launch_count["n"] += 2; L.check(lib.dle_cosine_rows_fwd(_ptr(x), _row_major_2d(x, "x"), _ptr(y), _row_major_2d(y, "y"), rows, H,
                                                              _ptr(ws[1:]), _ptr(ws), _stream()), "dle_cosine_rows_fwd")
    return ws[0]


def cosine_rows_bwd(x, y, grad_scale):
    """dx (bf16 [rows, H]) of cosine_rows_fwd's loss times grad_scale (fp32 device scalar)."""
    lib = L.load()
    rows, H = x.shape
    dx = torch.empty((rows, H), device=x.device, dtype=bf16)
    L.launch_count["n"] += 1; L.check(lib.dle_cosine_rows_bwd(_ptr(x), _row_major_2d(x, "x"), _ptr(y), _row_major_2d(y, "y"), rows, H,
                                                              _ptr(_req(grad_scale, torch.float32, "grad_scale")), _ptr(dx), H, _stream()),
                                      "dle_cosine_rows_bwd")
    return dx


def add_rows_bf16(dst, src, colsum=None):
    """dst += src (bf16 2-D views of one shape, fp32 add); colsum (fp32 [cols]) += column sums of src when given."""
    lib = L.load()
    _req(dst, bf16, "dst"); _req(src, bf16, "src")
    if dst.shape != src.shape:
        raise L.DleError(f"add_rows_bf16: shapes differ, {tuple(dst.shape)} and {tuple(src.shape)}")
    if colsum is not None:
        _req(colsum, torch.float32, "colsum")
    L.launch_count["n"] += 1; L.check(lib.dle_add_rows_bf16(_ptr(dst), _row_major_2d(dst, "dst"), _ptr(src), _row_major_2d(src, "src"),
                                                            dst.shape[0], dst.shape[1], _ptr(colsum), _stream()), "dle_add_rows_bf16")
