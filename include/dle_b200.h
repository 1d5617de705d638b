/* dle_b200.h -- C ABI of libdle_b200.so: hand-written sm_90a (H100) kernels for the BERT-large
 * pretraining hot path (NVIDIA/DeepLearningExamples, PyTorch/LanguageModeling/BERT).
 *
 * Conventions
 *  - plain pointers and sizes only; every pointer is a DEVICE pointer unless named host_*.
 *  - `stream` is a cudaStream_t passed as void*; kernels are enqueued, never synchronised.
 *  - no allocation in hot calls (the caller owns outputs and workspaces); the two *_plan_create
 *    functions allocate small device tables once.
 *  - return 0 on success; negative errno-style codes otherwise (DLE_ERR_*).  Nothing throws.
 *  - numeric overflow in gradients is NOT an error: it is reported through the device-side
 *    found_inf flag exactly like the reference's noop_flag protocol.
 *  - activations are bf16 row-major [tokens, features], tokens ordered b*S + s.
 *  - dropout: masks are regenerated, never stored.  Every dropout kernel takes a host `seed`, an RNG `dropout_stream` id (one per
 *    call site) and an optional DEVICE counter `seed_dev` (NULL = unused): the effective seed is seed + *seed_dev * 0x9E3779B97F4A7C15.
 *    The counter lets a captured CUDA graph (whose host arguments are frozen) draw fresh masks on every replay: bump it once per
 *    training step with dle_advance_u64 (the reference gets the same effect from the Philox offset of torch's graph-safe generator,
 *    run_pretraining.py:622-626).  Forward and backward of one step must see the same counter value.
 *
 * There is no C FFI in the reference for this path (SURVEY.md 8b); each entry point cites the
 * reference Python/C++ site it replaces (paths relative to PyTorch/LanguageModeling/BERT/).
 */
#ifndef DLE_B200_H
#define DLE_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DLE_ERR_INVALID (-22)
#define DLE_ERR_CUDA (-5)
#define DLE_ERR_NOSYS (-38)

#define DLE_DTYPE_F32 0
#define DLE_DTYPE_BF16 1

/* library / build identification: returns the compiled arch (90) and writes a version string */
int dle_version(char* host_buf, int host_buf_len);

/* ------------------------------------------------------------------------------------------
 * Dense GEMM with fused epilogue  (wgmma + TMA + mbarrier pipeline)
 *   D[M,N] = alpha * A[M,K] x B[N,K]^T  (+ epilogue)
 * replaces: F.linear -> cuBLAS at modeling.py:160 (LinearActivation), :345-347 (query/key/value),
 *   :395,:431 (dense), :553 (decoder) and their autograd dgrad/wgrad GEMMs; the bias+gelu
 *   (modeling.py:121-122,156-160) and dropout+residual (modeling.py:396-397,432-433) pointwise
 *   passes are epilogue modes.
 * layouts: DLE_LAYOUT_K  : operand stored row-major [rows, K]  (reduction dim contiguous)
 *          DLE_LAYOUT_MN : operand stored row-major [K, rows]  (M resp. N contiguous)
 *   forward  y = x W^T   : A = x  (K),  B = W  (K)
 *   dgrad   dx = dy W    : A = dy (K),  B = W  (MN)
 *   wgrad   dW = dy^T x  : A = dy (MN), B = x  (MN), epilogue ATOMIC_F32 with split-K
 * ------------------------------------------------------------------------------------------ */
#define DLE_LAYOUT_K 0
#define DLE_LAYOUT_MN 1

#define DLE_EPI_BIAS 0                  /* out = acc (+ bias[n])                        bf16 */
#define DLE_EPI_BIAS_GELU 1             /* out2 = u = acc + bias; out = gelu_tanh(u)    bf16 */
#define DLE_EPI_BIAS_DROPOUT_RESIDUAL 2 /* out = dropout(acc + bias) + aux              bf16 */
#define DLE_EPI_DGELU 3                 /* out = acc * gelu_tanh'(aux)                  bf16 */
#define DLE_EPI_ADD 4                   /* out = acc + aux                              bf16 */
#define DLE_EPI_ATOMIC_F32 5            /* out(fp32) += acc   (split-K, red.global.add)      */
#define DLE_EPI_F32 6                   /* out(fp32) = acc (+ bias)                          */
#define DLE_EPI_BIAS_TANH 7             /* out = tanh(acc + bias)   (pooler)            bf16 */
#define DLE_EPI_COUNT 8

typedef struct dle_gemm_args {
    const void* A;        /* bf16 */
    const void* B;        /* bf16 */
    void* out;            /* bf16 [M, ldo], or fp32 for DLE_EPI_ATOMIC_F32 / DLE_EPI_F32 */
    void* out2;           /* bf16 [M, ldo2]: pre-activation for DLE_EPI_BIAS_GELU, else NULL */
    const void* bias;     /* bf16 [N] or NULL */
    const void* aux;      /* bf16 [M, ld_aux]: residual / pre-activation, or NULL */
    int32_t M, N, K;
    int32_t a_layout, b_layout;
    int64_t lda, ldb, ldo, ldo2, ld_aux;   /* leading dimensions in elements */
    int32_t epilogue;
    int32_t splits;        /* split-K factor (DLE_EPI_ATOMIC_F32 only), 0/1 = none */
    int32_t tile_n;        /* 0 = auto (256), or 128 */
    float alpha;           /* scales the accumulator before the epilogue */
    float dropout_p;       /* DLE_EPI_BIAS_DROPOUT_RESIDUAL: drop probability, 0 = off */
    uint32_t dropout_stream; /* RNG stream id (distinct per call site so masks differ per layer) */
    uint64_t seed;
    const uint64_t* seed_dev; /* optional device step counter mixed into the seed (see Conventions), or NULL */
    void* colsum_out;      /* fp32 [N] or NULL: += column sums of the bf16 output (bias gradient of the producing layer), atomics */
} dle_gemm_args;

int dle_gemm_bf16(const dle_gemm_args* host_args, void* stream);

/* ------------------------------------------------------------------------------------------
 * Fused multi-head self-attention (tensor-core QK^T and PV, online softmax, in-kernel dropout);
 * the [B,A,S,S] score tensor never exists in HBM.
 * replaces: BertSelfAttention.forward modeling.py:349-376 (transpose_for_scores, bmm, /sqrt(d),
 *   + mask, softmax, dropout, bmm, transpose+contiguous) and its autograd backward.
 * qkv: bf16 [B*S, 3*A*64] (q | k | v column blocks, head h at columns h*64) -- the packed output
 *   of one QKV projection GEMM.   mask: fp32 additive [B, S] ((1-m)*-10000, modeling.py:864-872)
 *   or NULL.   ctx/dctx: bf16 [B*S, A*64].   lse: fp32 [B, A, S] (natural-log sum-exp of the
 *   scaled+masked scores, saved for backward).   head dim is fixed at 64; S % 128 == 0, S <= 512.
 * seq_first: 0 = token rows ordered b*S+s ([B,S,*]); 1 = s*B+b (the reference's [S,B,*] layer convention,
 *   modeling.py:330-338,498) -- both are read in place through 3-D TMA maps.
 * ------------------------------------------------------------------------------------------ */
int dle_attn_fwd(const void* qkv, const float* mask, void* ctx, float* lse, int32_t B, int32_t S, int32_t A,
                 int32_t seq_first, float dropout_p, uint64_t seed, const uint64_t* seed_dev, uint32_t dropout_stream, void* stream);
/* delta_ws: fp32 workspace [B, A, S] (row dots of dO and O); dqkv: bf16 [B*S, 3*A*64], fully overwritten (dQ, dK and dV are
 * each accumulated on chip by exactly one CTA: no atomics, bitwise reproducible);
 * dbias_qkv: fp32 [3*A*64] or NULL: += column sums of dqkv (the q/k/v bias gradients), must be zeroed by the caller */
int dle_attn_bwd(const void* qkv, const float* mask, const void* ctx, const void* dctx, const float* lse,
                 void* dqkv, float* delta_ws, float* dbias_qkv, int32_t B, int32_t S, int32_t A, int32_t seq_first, float dropout_p,
                 uint64_t seed, const uint64_t* seed_dev, uint32_t dropout_stream, void* stream);

/* ------------------------------------------------------------------------------------------
 * (bias +) dropout + residual-add + LayerNorm, vectorised warp-shuffle kernels (HBM-bound)
 * replaces: BertSelfOutput.forward / BertOutput.forward modeling.py:394-398,430-434
 *   (dropout -> `+ input_tensor` -> nn.LayerNorm(eps=1e-12)), BertPredictionHeadTransform :534.
 *   z = dropout(x + bias) + residual   (bias, residual optional; skip when the GEMM epilogue
 *                                       already produced z)
 *   y = (z - mean) * rstd * gamma + beta ; mean/rstd fp32 [T] saved for backward.
 * H % 256 == 0, H <= 1024.  z_out may be NULL when no bias/dropout/residual is applied (z == x).
 * ------------------------------------------------------------------------------------------ */
int dle_add_ln_fwd(const void* x, const void* bias, const void* residual, const void* gamma, const void* beta,
                   void* z_out, void* y, float* mean, float* rstd, int64_t T, int32_t H, float eps,
                   float dropout_p, uint64_t seed, const uint64_t* seed_dev, uint32_t dropout_stream, void* stream);
/* backward: dz = dLN(dy); dx = dropout_bwd(dz) written to dx_out when dropout_p > 0 (else dx == dz
 * and dx_out may be NULL).  dz is also the gradient of the residual branch.  Column reductions are written as fp32 partials [n_part, H] into the caller's workspace:
 *   part_dgamma, part_dbeta, part_dbias (sum_t dx).  n_part = dle_ln_bwd_partials(T).  A second
 *   call dle_colsum_finalize reduces them to bf16/fp32 gradients. */
int dle_ln_bwd_partials(int64_t T);             /* upper bound over H (workspace sizing) */
int dle_ln_bwd_partials_h(int64_t T, int32_t H); /* rows of partials actually written for this H */
int dle_add_ln_bwd(const void* dy, const void* z, const float* mean, const float* rstd, const void* gamma,
                   void* dz_out, void* dx_out, float* part_dgamma, float* part_dbeta, float* part_dbias,
                   int64_t T, int32_t H, float dropout_p, uint64_t seed, const uint64_t* seed_dev, uint32_t dropout_stream, void* stream);
/* out[n] = sum_p part[p, n]; out dtype DLE_DTYPE_BF16 or DLE_DTYPE_F32; accumulate != 0 adds to out */
int dle_colsum_finalize(const float* part, int32_t n_part, int32_t N, void* out, int32_t out_dtype,
                        int32_t accumulate, void* stream);
/* n_arrays stacked partial sets part[a][p][n] -> out[a][n] in ONE launch (dgamma, dbeta, dbias of a LayerNorm) */
int dle_colsum_finalize_batched(const float* part, int32_t n_arrays, int32_t n_part, int32_t N, void* out,
                                int32_t out_dtype, int32_t accumulate, void* stream);
/* column sum of a bf16 matrix [T, N] (bias gradients): part = fp32 [dle_colsum_partials(T), N] */
int dle_colsum_partials(int64_t T);
int dle_colsum_bf16(const void* x, int64_t T, int32_t N, int64_t ldx, float* part, void* stream);

/* ------------------------------------------------------------------------------------------
 * bias + tanh-GELU, standalone vectorised kernels (the GEMM epilogue modes DLE_EPI_BIAS_GELU /
 * DLE_EPI_DGELU are the fused forms).
 * replaces: LinearActivation.forward's act_fn(linear + bias) modeling.py:121-122,156-160.
 *   fwd: u_out (optional) = x + bias ; y = gelu_tanh(u)       bwd: du = dy * gelu_tanh'(u)
 * ------------------------------------------------------------------------------------------ */
int dle_bias_gelu_fwd(const void* x, const void* bias, void* u_out, void* y, int64_t T, int32_t N, void* stream);
int dle_bias_gelu_bwd(const void* dy, const void* u, void* du, int64_t T, int32_t N, void* stream);

/* ------------------------------------------------------------------------------------------
 * Embedding gathers + sum + LayerNorm (+ dropout)
 * replaces: BertEmbeddings.forward modeling.py:285-301 (3 nn.Embedding gathers with int64 indices,
 *   add, LayerNorm, dropout).  The gathers are integer work: rows are fetched bit-exactly.
 *   z_out: bf16 [B*S, H] pre-LN sum (saved for backward).  Out-of-range ids set *err_flag (int32
 *   device flag, may be NULL) instead of faulting.
 * bwd: dz = dLN(dropout_bwd(dy)); scatter-add dz rows into fp32 gradient tables
 *   (dword [V,H], dpos [P,H], dtype [2,H]) with red.global.add; dgamma/dbeta partials as above.
 * ------------------------------------------------------------------------------------------ */
int dle_embed_ln_fwd(const int64_t* input_ids, const int64_t* token_type_ids, const void* word, const void* pos,
                     const void* type, const void* gamma, const void* beta, void* z_out, void* y, float* mean,
                     float* rstd, int32_t B, int32_t S, int32_t H, int32_t V, int32_t P, int32_t NT, float eps,
                     float dropout_p, uint64_t seed, const uint64_t* seed_dev, uint32_t dropout_stream, int32_t* err_flag, void* stream);
int dle_embed_ln_bwd(const void* dy, const void* z, const float* mean, const float* rstd, const void* gamma,
                     const int64_t* input_ids, const int64_t* token_type_ids, float* dword, float* dpos,
                     float* dtype_tab, float* part_dgamma, float* part_dbeta, int32_t B, int32_t S, int32_t H,
                     float dropout_p, uint64_t seed, const uint64_t* seed_dev, uint32_t dropout_stream, void* stream);
/* masked-row gather (dense sequence output): out[i,:] = x[idx[i],:]  -- bit exact.
 * replaces torch.index_select at modeling.py:590.  bwd scatters rows back (rows are unique).
 * idx[i] == -1 marks a PADDING slot of a static-size index list (torch.nonzero_static): gather writes a zero row, scatter skips it;
 * any other out-of-range index sets *err_flag (gather) / is skipped (scatter). */
int dle_gather_rows(const void* x, const int64_t* idx, void* out, int64_t n_idx, int32_t H, int64_t n_rows,
                    int32_t* err_flag, void* stream);
int dle_scatter_rows(const void* dy, const int64_t* idx, void* dx, int64_t n_idx, int32_t H, int64_t n_rows,
                     void* stream);
/* ------------------------------------------------------------------------------------------
 * Softmax cross-entropy over the vocabulary on bf16 logits, fp32 arithmetic, one pass per direction (HBM-bound).
 * replaces: CrossEntropyLoss(ignore_index=-1) on the MLM prediction scores, run_pretraining.py:85-95 (under the reference's autocast:
 *   an fp32 copy of the [rows, V] logits + log_softmax + nll_loss and their backward).
 *   fwd: lse[r] = logsumexp_v logits[r,v]; loss_rows[r] = lse[r] - logits[r, labels[r]], 0 where labels[r] == ignore_index.
 *        (mean loss = sum(loss_rows) / #counted rows: two tiny reductions left to the caller).  A label outside [0,V) that is
 *        not ignore_index sets *err_flag (may be NULL).  V % 8 == 0, V <= 32768.
 *   bwd: dlogits[r,v] = (softmax(logits[r])[v] - [v == labels[r]]) * *grad_scale for counted rows, 0 otherwise; grad_scale is a DEVICE
 *        fp32 scalar (dLoss / #counted rows) so no host value is needed.  dlogits may alias logits.
 * ------------------------------------------------------------------------------------------ */
int dle_softmax_ce_fwd(const void* logits, const int64_t* labels, float* lse, float* loss_rows, int64_t rows, int32_t V,
                       int64_t ld, int64_t ignore_index, int32_t* err_flag, void* stream);
int dle_softmax_ce_bwd(const void* logits, const int64_t* labels, const float* lse, const float* grad_scale, void* dlogits,
                       int64_t rows, int32_t V, int64_t ld, int64_t ld_d, int64_t ignore_index, void* stream);

/* *counter += delta on the stream (one thread): the per-step bump of a dropout `seed_dev` counter; graph-capturable */
int dle_advance_u64(uint64_t* counter, uint64_t delta, void* stream);
/* fp32 -> bf16 conversion (gradient tables, weight casts); bf16 -> fp32 */
int dle_cast_f32_to_bf16(const float* x, void* y, int64_t n, void* stream);
int dle_cast_bf16_to_f32(const void* x, float* y, int64_t n, void* stream);

/* ------------------------------------------------------------------------------------------
 * Multi-tensor LAMB: the whole optimizer step over all parameter tensors in 3 launches
 * (grad-norm/found_inf/step++, stage 1, stage 2) driven by a device-resident tensor table.
 * replaces: FusedLAMBAMP.step lamb_amp_opt/fused_lamb/fused_lamb.py:130-260 and the pybind module
 *   fused_lamb_CUDA.{multi_tensor_l2norm, multi_tensor_lamb} (lamb_amp_opt/csrc/frontend.cpp:28-33,
 *   multi_tensor_lamb.cu:371-500, multi_tensor_l2norm_kernel.cu:153-216), ~100 launches there.
 * Semantics kept: grads arrive scaled by *scale; found_inf => nothing is updated and `step` is not
 *   incremented; global-norm clipping against max_grad_norm*scale; per-tensor trust ratio only for
 *   weight_decay != 0 (or use_nvlamb); bias correction from the device-side int32 step;
 *   optional 16-bit model copy written with the fp32 master (5-list form).
 * ------------------------------------------------------------------------------------------ */
typedef struct dle_lamb_tensor {
    void* grad;          /* grad_dtype, numel elements (scaled by the loss scale) */
    float* param;        /* fp32 parameter / fp32 master copy, updated in place   */
    float* exp_avg;      /* fp32 */
    float* exp_avg_sq;   /* fp32 */
    void* model_param;   /* bf16 model copy written alongside, or NULL            */
    int64_t numel;
    int32_t group;       /* index into the group array                            */
    int32_t reserved;
} dle_lamb_tensor;

typedef struct dle_lamb_group {
    const float* lr;     /* device fp32 scalar  (fused_lamb.py:23) */
    int32_t* step;       /* device int32 scalar (fused_lamb.py:24), incremented unless found_inf */
    float beta1, beta2, eps, weight_decay;
    int32_t bias_correction, grad_averaging;
} dle_lamb_group;

/* builds the device tensor/chunk tables (one cudaMalloc + copy); *plan_out is an opaque handle */
int dle_lamb_plan_create(const dle_lamb_tensor* host_tensors, int32_t n_tensors, const dle_lamb_group* host_groups,
                         int32_t n_groups, int32_t grad_dtype, void** plan_out);
int dle_lamb_plan_destroy(void* plan);
/* re-point the plan at new grad/param addresses (same tensor count, sizes, groups): one small async H2D copy from a pinned staging
 * ring owned by the plan -- no allocation and no host synchronisation on the per-step path, and legal while `stream` is being captured
 * into a CUDA graph (at most 4 captured updates per plan: DLE_ERR_NOSYS beyond that) */
int dle_lamb_plan_update(void* plan, const dle_lamb_tensor* host_tensors, int32_t n_tensors, void* stream);
/* scale: device fp32 loss scale or NULL (=1).  found_inf_out / global_grad_norm_out: device fp32
 * scalars written by the call (global_grad_norm is the norm of the SCALED grads, as in the reference).
 * per_tensor_norms_out: optional device fp32 [2*n_tensors] (param norms then update norms). */
int dle_lamb_step(void* plan, const float* scale, float max_grad_norm, int32_t adam_w_mode, int32_t use_nvlamb,
                  float* found_inf_out, float* global_grad_norm_out, float* per_tensor_norms_out, void* stream);
/* Multi-tensor Adam / AdamW (+ global-norm clipping) on a plan built by dle_lamb_plan_create (the group's `grad_averaging`
 * is ignored; `bias_correction` selects 1-beta^t corrections).  max_grad_norm <= 0 disables clipping; clip_eps = 1e-6 reproduces
 * the SQuAD GradientClipper's coef = max/(norm + 1e-6).
 * replaces: apex.optimizers.FusedAdam(..., bias_correction=False) + GradientClipper (amp_C.multi_tensor_l2norm / multi_tensor_scale)
 *   at run_squad.py:703-724,969-975,1092-1099.  Two launches: grad pass + one fused apply pass. */
int dle_adam_step(void* plan, const float* scale, float max_grad_norm, float clip_eps, int32_t adam_w_mode,
                  float* found_inf_out, float* global_grad_norm_out, void* stream);
/* standalone multi-tensor L2 norm over the plan's gradients (fused_lamb_CUDA.multi_tensor_l2norm) */
int dle_lamb_grad_norm(void* plan, float* norm_out, float* found_inf_out, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* DLE_B200_H */
