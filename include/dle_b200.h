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
#define DLE_EPI_BIAS_GELU 1             /* out2 = u = acc + bias; out = gelu_tanh(u)    bf16 (out2 NULL: u not stored) */
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
    void* out2;           /* bf16 [M, ldo2]: pre-activation for DLE_EPI_BIAS_GELU (or NULL), else NULL */
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
/* packed variable-length forward (inference): qkv [T, 3*A*64], ctx [T, A*64], cu_seqlens int32 [B+1] (device, non-decreasing,
 * cu_seqlens[0] == 0), every length <= max_seqlen <= 512.  No mask, no dropout, no lse.  Sequence b is token rows
 * cu_seqlens[b] .. cu_seqlens[b+1]; it attends to its own rows only, and only those rows of ctx are written.  A length above
 * max_seqlen is clamped to max_seqlen; a length of 0 is legal.  A valid row gets the bits dle_attn_fwd gives it in a padded
 * batch with a -10000 mask on the padding. */
int dle_attn_fwd_varlen(const void* qkv, const int32_t* cu_seqlens, void* ctx, int32_t B, int32_t max_seqlen, int32_t A, void* stream);
/* packed variable-length forward for training: dle_attn_fwd_varlen plus dle_attn_fwd's dropout, and lse fp32 [A, T] (head h, token
 * row t at h*T + t; rows outside every sequence are not written).  cu_seqlens[B] <= T.  The Philox block of (sequence b, head h,
 * in-sequence query q, in-sequence key k) is drawn at ((b*A + h)*drop_stride + q)*drop_stride + k, drop_stride a multiple of 64 with
 * max_seqlen <= drop_stride <= 512: with drop_stride = S a right-padded batch draws dle_attn_fwd's keep bits, and a valid row gets
 * dle_attn_fwd's bits (ctx and lse) under a -10000 mask on the padding. */
int dle_attn_fwd_varlen_train(const void* qkv, const int32_t* cu_seqlens, void* ctx, float* lse, int32_t T, int32_t B,
                              int32_t max_seqlen, int32_t A, int32_t drop_stride, float dropout_p, uint64_t seed,
                              const uint64_t* seed_dev, uint32_t dropout_stream, void* stream);
/* delta_ws: fp32 workspace [B, A, S] (row dots of dO and O); dqkv: bf16 [B*S, 3*A*64], fully overwritten (dQ, dK and dV are
 * each accumulated on chip by exactly one CTA: no atomics, bitwise reproducible);
 * dbias_qkv: fp32 [3*A*64] or NULL: += column sums of dqkv (the q/k/v bias gradients), must be zeroed by the caller */
int dle_attn_bwd(const void* qkv, const float* mask, const void* ctx, const void* dctx, const float* lse,
                 void* dqkv, float* delta_ws, float* dbias_qkv, int32_t B, int32_t S, int32_t A, int32_t seq_first, float dropout_p,
                 uint64_t seed, const uint64_t* seed_dev, uint32_t dropout_stream, void* stream);
/* packed variable-length backward: the arguments of dle_attn_fwd_varlen_train, with delta_ws fp32 [A, T].  Only the rows of dqkv
 * inside a sequence are written (each by exactly one CTA, as in dle_attn_bwd), and dbias_qkv (zeroed by the caller, or NULL) receives
 * the column sums of those rows only.  With drop_stride = S, the valid rows of a right-padded batch get dle_attn_bwd's bits when dctx
 * is 0 on the padding. */
int dle_attn_bwd_varlen(const void* qkv, const int32_t* cu_seqlens, const void* ctx, const void* dctx, const float* lse,
                        void* dqkv, float* delta_ws, float* dbias_qkv, int32_t T, int32_t B, int32_t max_seqlen, int32_t A,
                        int32_t drop_stride, float dropout_p, uint64_t seed, const uint64_t* seed_dev, uint32_t dropout_stream,
                        void* stream);

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
 * position_ids: int64 [B*S] or NULL.  NULL reads position s = row % S (modeling.py:285-301 builds arange(S) per row); otherwise
 *   the position of token row r is position_ids[r] (packed samples restart at 0).  Dropout stays keyed by element index, so
 *   position_ids = arange(S) per row gives the NULL path's bits.  The forward treats a position outside [0, P) like an out-of-range
 *   id (sets *err_flag, reads row 0); the backward takes the forward's ids and positions as they are.
 * ------------------------------------------------------------------------------------------ */
int dle_embed_ln_fwd(const int64_t* input_ids, const int64_t* token_type_ids, const void* word, const void* pos,
                     const void* type, const void* gamma, const void* beta, void* z_out, void* y, float* mean,
                     float* rstd, int32_t B, int32_t S, int32_t H, int32_t V, int32_t P, int32_t NT, float eps,
                     float dropout_p, uint64_t seed, const uint64_t* seed_dev, uint32_t dropout_stream, int32_t* err_flag, void* stream,
                     const int64_t* position_ids);
int dle_embed_ln_bwd(const void* dy, const void* z, const float* mean, const float* rstd, const void* gamma,
                     const int64_t* input_ids, const int64_t* token_type_ids, float* dword, float* dpos,
                     float* dtype_tab, float* part_dgamma, float* part_dbeta, int32_t B, int32_t S, int32_t H,
                     float dropout_p, uint64_t seed, const uint64_t* seed_dev, uint32_t dropout_stream, void* stream,
                     const int64_t* position_ids);
/* segment table of a packed batch (several samples per row; replaces the position ids of modeling.py:285-301 and the [CLS] row the
 * pooler reads at modeling.py:518-523).  mask: int64 [B, S], the sample number of each token: the j-th sample of a row (1 <= j <= k)
 * holds j, samples are contiguous and increasing, and the row's padding tail holds 0 and comes last.  Outputs, all static in size:
 *   cu_seqlens   int32 [B*(k+1) + 1]: row b owns sequences b*(k+1) .. b*(k+1)+k; sequence b*(k+1)+j-1 is sample j (length 0 when the
 *                row has fewer than j samples) and b*(k+1)+k is the row's padding tail.  A row's lengths sum to S, so every token lies in
 *                exactly one sequence and row b starts at b*S.
 *   position_ids int64 [B*S]: index of the token inside its sample (inside the tail for tail tokens).
 *   cls_index    int64 [B*k]: b*S + start of sample j at b*k + j-1, or -1 when the row has no sample j (dle_gather_rows: a zero row).
 * A malformed row (a value outside 0..k, a decrease, a skipped number, a non-zero value after a 0) sets *err_flag (may be NULL) and is
 * written as one tail segment of length S with positions 0..S-1 and no samples.  One warp per row, no host work: graph-capturable.
 * B*(k+1) <= 65535. */
int dle_segment_table(const int64_t* mask, int32_t B, int32_t S, int32_t k, int32_t* cu_seqlens, int64_t* position_ids,
                      int64_t* cls_index, int32_t* err_flag, void* stream);
/* per-sample span logits of a packed SQuAD batch (several features per row; serves the split of the QA head's logits at
 * modeling.py:1366-1369 and the span cross-entropy over them at run_squad.py:1066-1079, which must see one feature per row).
 *   unpack:    logits [B*S, 2] with row stride ld (column 0 start, column 1 end) on the packed grid, and cu_seqlens of
 *              dle_segment_table for the same B, S, k.  Slot b*k + j-1 holds sample j of row b (sequence b*(k+1) + j-1):
 *              start_out[b*k + j-1, p] = logits[cu + p, 0] for p < len, and fill for len <= p < S and across an empty slot;
 *              end_out likewise from column 1.  start_out, end_out: [B*k, S], contiguous.
 *   pack_grad: the inverse for the gradients: dlogits[cu + p] = (dstart[slot, p], dend[slot, p]) for every sample token, and exactly
 *              (0, 0) at every tail token.  Every row of dlogits is written once (no memset needed).
 * Both only move values: bit exact.  dtype DLE_DTYPE_BF16 or DLE_DTYPE_F32 for every tensor (fill is rounded to it).  No host work:
 * graph-capturable.  A malformed row is one tail segment in the table, so all its slots come out as fill.  B*(k+1) <= 65535. */
int dle_span_logits_unpack(const void* logits, int64_t ld, const int32_t* cu_seqlens, int32_t B, int32_t S, int32_t k,
                           int32_t dtype, float fill, void* start_out, void* end_out, void* stream);
int dle_span_logits_pack_grad(const void* dstart, const void* dend, const int32_t* cu_seqlens, int32_t B, int32_t S, int32_t k,
                              int32_t dtype, void* dlogits, int64_t ld, void* stream);
/* sequence-classification head: dropout of the pooled rows, then the [H] -> [L] classifier (modeling.py:1145-1155, the
 * BertForSequenceClassification forward whose logits run_glue.py:631-634 feeds to CrossEntropyLoss).  L is too narrow for the GEMM.
 *   fwd: x [R, H] bf16 (row stride ldx, a multiple of 8, 16-byte aligned), W [L, H] bf16 contiguous (16-byte aligned), b [L] ->
 *        logits [R, L] contiguous:  logits[r, l] = sum_c x[r,c] * keep[r,c] * scale * W[l,c] + b[l], fp32 accumulation in a fixed
 *        order per row (a row's logits depend on that row alone), rounded once.
 *   bwd: dlogits [R, L] contiguous -> dx [R, H] bf16 contiguous, dx[r,c] = keep[r,c] * scale * sum_l dlogits[r,l] * W[l,c];
 *        dW [L, H] and db [L]: fp32 sums over rows, per-slab partials in `part` (dle_cls_head_bwd_partials(R) * L * (H + 1) floats)
 *        summed in a fixed order by the colsum finalize kernel -- deterministic, no atomics; a row whose dlogits are 0 adds exactly 0.
 *        The keep bits are recomputed (nothing is stored), so backward sees forward's mask.
 * keep[r,c] is the hidden-dropout bit of flat element r*H + c under (seed, dropout_stream), as at every other hidden-dropout site
 * (dropout_keep8 of common.cuh, the step counter seed_dev mixed in when non-NULL), scale = 1/(1-p); p = 0 keeps everything.
 * dtype (DLE_DTYPE_BF16 or DLE_DTYPE_F32) is that of b, logits, dlogits, dW and db: the parameter dtype.  1 <= L <= 32, H % 32 == 0,
 * 1 <= R <= 2097120, 0 <= p < 1; anything else returns DLE_ERR_INVALID before any CUDA call.  No host work: graph-capturable. */
int dle_cls_head_fwd(const void* x, int64_t ldx, const void* w, const void* b, int32_t R, int32_t H, int32_t L, int32_t dtype,
                     float dropout_p, uint64_t seed, const uint64_t* seed_dev, uint32_t dropout_stream, void* logits, void* stream);
int dle_cls_head_bwd_partials(int32_t R);
int dle_cls_head_bwd(const void* dlogits, const void* x, int64_t ldx, const void* w, int32_t R, int32_t H, int32_t L, int32_t dtype,
                     float dropout_p, uint64_t seed, const uint64_t* seed_dev, uint32_t dropout_stream, void* dx, float* part,
                     void* dw, void* db, void* stream);
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

/* ------------------------------------------------------------------------------------------
 * General distillation losses (MiniLM / TinyBERT backbone distillation), without the [B, A, S, S] tensors.
 *
 * Relation-KL: per (b, h) the student logits s = scale_s * X_s Y_s^T (+ mask_s) and teacher logits t = scale_t * X_t Y_t^T (+ mask_t),
 * each [S, S]; with where_rule != 0 every logit <= -100 (masked keys included) becomes 0 first.
 *   loss = norm * sum over the B*A*S query rows of KL(softmax(t) || softmax(s))
 * X / Y point at the 64 columns of head 0 in token-row matrices with row strides ld_s / ld_t (head h is 64*h columns further);
 * token row of (b, s) = b*S + s, or s*B + b when seq_first.  Head dim 64, S % 64 == 0, S <= 512.
 *   attention scores : X = Q, Y = K (column blocks 0 and A of the packed qkv), mask, where_rule = 1
 *   value relation   : X = Y = ctx, no mask, where_rule = 0, scale = 1/sqrt(64)
 * replaces: TransformerLosses.compute_loss / compute_loss_ with attention_loss = value_state_loss = "kld"
 *   distillation/losses.py:37-61,77-88 (torch.where, bmm, LogSoftmax, Softmax, KLDivLoss(batchmean) / (A*S)) and the score tensor
 *   modeling.py:298-300,378-383 it reads.
 * fwd: lse_s / lse_t fp32 [B, A, S] for backward; partial fp32 [dle_relkl_partials(B, S, A)] workspace; loss fp32 [1].  Partials are
 *   summed in a fixed order (no atomics): bitwise reproducible and graph-capturable.
 * bwd: dS = grad_scale[0] * norm * scale_s * (p_s - p_t), 0 where the where rule substituted; dx = dS Y_s, dy = dS^T X_s (bf16, row
 *   stride ld_d, head-0 column block).  dx == dy (X = Y) adds dS^T X_s onto dS Y_s.  dzero (or NULL): a head-0 column block that is
 *   zero-filled (the V block of a packed qkv gradient). */
int dle_relkl_partials(int32_t B, int32_t S, int32_t A);
int dle_relkl_fwd(const void* xs, const void* ys, const void* xt, const void* yt, int64_t ld_s, int64_t ld_t, const float* mask_s,
                  const float* mask_t, float scale_s, float scale_t, int32_t where_rule, int32_t B, int32_t S, int32_t A, int32_t seq_first,
                  float norm, float* lse_s, float* lse_t, float* partial, float* loss, void* stream);
int dle_relkl_bwd(const void* xs, const void* ys, const void* xt, const void* yt, int64_t ld_s, int64_t ld_t, const float* mask_s,
                  const float* mask_t, float scale_s, float scale_t, int32_t where_rule, int32_t B, int32_t S, int32_t A, int32_t seq_first,
                  const float* lse_s, const float* lse_t, const float* grad_scale, float norm, void* dx, void* dy, void* dzero,
                  int64_t ld_d, void* stream);
/* Cosine rows: loss = mean over rows of 1 - <x, y> / sqrt((|x|^2 + 1e-12)(|y|^2 + 1e-12)) on bf16 rows [rows, H], fp32 arithmetic.
 * replaces: CosineEmbeddingLoss()(pred.view(-1, H), target.view(-1, H), 1), distillation/losses.py:63-70 (hidden / embedding states).
 * fwd: partial fp32 [dle_cosine_rows_partials(rows)] workspace, loss fp32 [1], fixed-order sums.  bwd: dx (bf16) = grad_scale[0] *
 * d loss / dx; no gradient for y (the teacher). */
int dle_cosine_rows_partials(int64_t rows);
int dle_cosine_rows_fwd(const void* x, int64_t ldx, const void* y, int64_t ldy, int64_t rows, int32_t H, float* partial, float* loss,
                        void* stream);
int dle_cosine_rows_bwd(const void* x, int64_t ldx, const void* y, int64_t ldy, int64_t rows, int32_t H, const float* grad_scale,
                        void* dx, int64_t ldd, void* stream);
/* dst[r, c] += src[r, c] on bf16 [rows, cols] (fp32 add, one rounding); colsum (fp32 [cols] or NULL) += column sums of src, atomics.
 * Folds a distillation loss's gradient of an encoder layer's qkv into the layer's own before its QKV dgrad (the loss term of the
 * q / k bias gradients, BertSelfAttention.query / key in modeling.py:298-300). */
int dle_add_rows_bf16(void* dst, int64_t ld_dst, const void* src, int64_t ld_src, int64_t rows, int32_t cols, float* colsum,
                      void* stream);

#ifdef __cplusplus
}
#endif
#endif /* DLE_B200_H */
