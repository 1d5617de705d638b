// Fused multi-head self-attention for sm_90a (head dim 64, S in {128,256,384,512}) on warpgroup MMA (wgmma.mma_async m64n64k16,
// bf16 in, fp32 accumulators in registers).  Tiles of 64 rows x 64 bf16 (128-byte rows) are streamed into 1024-byte aligned,
// 128B-swizzled shared memory by cp.async double buffering and read there by wgmma as K-major or (through the transpose bit)
// MN-major operands; the P / dS operands go to wgmma from registers.
//
// Forward : one CTA per (batch, head, 128-query tile), two warpgroups x 64 query rows.  K / V come in 64-key tiles.
//           S = Q K^T, online softmax in registers, dropout (Philox, regenerated in backward), O += P V with P taken straight
//           from the S accumulators (as bf16 hi + lo parts).  The [B,A,S,S] score tensor the reference materialises 3x per layer
//           never exists in HBM.
// Varlen  : the forward over packed sequences (cu_seqlens, any length up to 512); each sequence visits only its own key tiles.  The
//           inference instance has no mask, no dropout and no lse; the training instance adds the forward's dropout and an lse [A, T].
// Backward: two kernels that recompute P from the saved log-sum-exp, so that every output is accumulated on chip by exactly
//           one CTA -- no atomics on dQ / dK / dV, deterministic:
//             dK / dV : one CTA (one warpgroup) per (batch, head, 64-key tile) walks the query tiles, computing S^T = K Q^T and
//                       dP^T = V dO^T, then dV += P~^T dO, dK += dS^T Q.
//             dQ      : one CTA (one warpgroup) per (batch, head, 64-query tile) walks the key tiles, computing S and dP again,
//                       then dQ += dS K.
//           Both are templated on the addressing: a padded [B, S] grid, or packed sequences (each CTA walks only its sequence's
//           ceil(len/64) tiles; rows past len are zero-filled, masked out of P and never stored).
// Dropout keying: the Philox block of (sequence b, head h, query q, key k) is ((b*A + h)*stride + q)*stride + k (>> 5), stride = S on
//          the padded grid and the caller's drop_stride for packed sequences -- with drop_stride = S a right-padded batch draws the
//          padded kernels' keep bits.
// Dropout: each Philox block (one query row x 32 keys) a CTA needs is computed by one thread, while the tile's score MMAs run,
//          and handed to the threads that apply it through shared memory.
//
// replaces BertSelfAttention.forward, PyTorch/LanguageModeling/BERT/modeling.py:349-376
// (transpose_for_scores, bmm, /sqrt(d), +mask, softmax, dropout, bmm, transpose+contiguous) and autograd.
#include "common.cuh"
#include "../../include/dle_b200.h"

namespace dle {

constexpr int HD = 64;                 // head dim
constexpr int KT = 64;                 // key / query tile of the loops
constexpr int TILE64_BYTES = KT * HD * 2;      // 8 KB: one [64 x 64] bf16 tile (128 B rows)
constexpr float LOG2E = 1.4426950408889634f;
constexpr float LN2 = 0.6931471805599453f;

__device__ __forceinline__ float ex2(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
// byte offset of 16-byte unit `ch` (8 bf16) of row r in a tile of 128-byte rows, XOR-swizzled by row % 8.  In a 1024-byte aligned
// tile this is exactly the hardware's 128-byte swizzle, which wgmma descriptors of mode SWIZZLE_128B read.
__device__ __forceinline__ uint32_t sw(int r, int ch) { return (uint32_t)(r * 128 + ((ch ^ (r & 7)) << 4)); }

struct AttnParams {
    const bf16* qkv;       // [T, 3H]
    const bf16* dctx;      // [T, H]      (backward)
    const float* mask;     // [B,S] additive or null
    const float* lse;      // [B,A,S]     (written by forward, read by backward)
    const float* delta;    // [B,A,S]     (backward)
    float* lse_out;
    bf16* ctx;             // [T, H]      (forward)
    bf16* dqkv;            // [T, 3H]     (backward)
    float* dbias;          // [3H] fp32 or null: += column sums of dqkv
    int B, S, A, H;
    int tok_stride_s, tok_stride_b;   // token row of (b, s) = b*tok_stride_b + s*tok_stride_s
    float scale, scale_log2;          // 1/sqrt(d), and that times log2(e)
    uint32_t drop_k2;                 // attn_dropout_k2(thresh15); dropout off when drop_on == 0
    uint32_t drop_on; float drop_scale; uint32_t drop_stream; unsigned long long seed; const unsigned long long* seed_dev;
    // packed sequences (backward kernels' VARLEN instances): sequence b is token rows cu_seqlens[b] .. cu_seqlens[b+1]; lse and
    // delta are [A, T]; S above is unused
    const int* cu_seqlens;
    int T, max_seqlen, drop_stride;
};

__device__ __forceinline__ long long tok_row(const AttnParams& p, int b, int s) {
    return (long long)b * p.tok_stride_b + (long long)s * p.tok_stride_s;
}
// the token rows of packed sequence b: row0 .. row0 + len, len clamped to [0, max_seqlen]
struct SeqRows { long long row0; int len; };
__device__ __forceinline__ SeqRows seq_rows(const int* cu_seqlens, int b, int max_seqlen) {
    const long long row0 = cu_seqlens[b];
    return SeqRows{row0, max(0, min(cu_seqlens[b + 1] - (int)row0, max_seqlen))};
}
// rows [s0, s0 + ROWS) of the 64-column block `col` of a [T, ld] bf16 matrix -> swizzled smem tile (cp.async, NT threads)
template <int ROWS, int NT>
__device__ __forceinline__ void load_tile(uint32_t dst, const bf16* base, long long ld, int col, const AttnParams& p, int b, int s0) {
#pragma unroll
    for (int i = 0; i < ROWS * 8 / NT; ++i) {
        const int idx = threadIdx.x + i * NT, r = idx >> 3, ch = idx & 7;
        cp_async16(dst + sw(r, ch), base + tok_row(p, b, s0 + r) * ld + col + ch * 8);
    }
}
// rows [s0, s0 + ROWS) of a sequence of `len` rows starting at token row `row0`, 64-column block `col` -> swizzled smem tile.  Rows at
// or past len are zero-filled; their source address is clamped to row0 (len >= 1 here), so no other sequence's row is read.
template <int ROWS, int NT>
__device__ __forceinline__ void load_tile_varlen(uint32_t dst, const bf16* base, long long ld, int col, long long row0, int len, int s0) {
#pragma unroll
    for (int i = 0; i < ROWS * 8 / NT; ++i) {
        const int idx = threadIdx.x + i * NT, r = idx >> 3, ch = idx & 7;
        const bool in = s0 + r < len;
        cp_async16_zfill(dst + sw(r, ch), base + (row0 + (in ? s0 + r : 0)) * ld + col + ch * 8, in ? 16u : 0u);
    }
}
// the backward kernels' tile load in either addressing mode
template <bool VARLEN, int ROWS, int NT>
__device__ __forceinline__ void load_rows(uint32_t dst, const bf16* base, long long ld, int col, const AttnParams& p, int b,
                                          const SeqRows& sr, int s0) {
    if constexpr (VARLEN) load_tile_varlen<ROWS, NT>(dst, base, ld, col, sr.row0, sr.len, s0);
    else load_tile<ROWS, NT>(dst, base, ld, col, p, b, s0);
}
// the cp.async groups up to the newest-but-N are in shared memory and visible to wgmma (async proxy) in every thread of the CTA
template <int N> __device__ __forceinline__ void tiles_ready() {
    cp_async_wait<N>();
    fence_proxy_async_smem();
    __syncthreads();
}
// acc[64 x 64] = A * T^T, A = 64 rows of 64 columns at `a` (K-major), T = 64 rows (the n dimension) of 64 columns at `t` (K-major).
// Issued only: the caller fences, commits and waits.
__device__ __forceinline__ void wg_abt(float (&acc)[8][4], uint32_t a, uint32_t t) {
#pragma unroll
    for (int kk = 0; kk < 4; ++kk)
        wgmma_m64n64k16<0, 0>(acc, make_wgmma_desc_sw128(a + kk * 32, 16, 1024), make_wgmma_desc_sw128(t + kk * 32, 16, 1024), kk > 0 ? 1u : 0u);
}
// acc[64 x 64] += A * T, A = packed bf16 accumulator pairs (pr[j][0]: row r, pr[j][1]: row r + 8 of column block j) and tile T
// holding 64 rows (the k dimension) of 64 columns (the n dimension), read MN-major.  Issued only.
__device__ __forceinline__ void wg_pt(float (&acc)[8][4], const uint32_t (&pr)[8][2], uint32_t t) {
#pragma unroll
    for (int kk = 0; kk < 4; ++kk)
        wgmma_m64n64k16_rs<1>(acc, pr[2 * kk][0], pr[2 * kk][1], pr[2 * kk + 1][0], pr[2 * kk + 1][1],
                              make_wgmma_desc_sw128(t + kk * 16 * 128, TILE64_BYTES, 1024));
}
// Row-major dropout (forward, dQ): a warp owns 16 query rows; per 64-key tile it needs the Philox blocks of its 16 rows x 2 key
// groups.  Lane l computes the block of row (first + l % 16), group l / 16 into slot l of the warp's 512-byte area; after __syncwarp
// the four lanes of a quad read the blocks of their rows r and r + 8 (broadcast).  drop_row = (bh*S + first row of the warp)*S.
__device__ __forceinline__ void warp_drop_blocks(uint4* slots, unsigned long long seed, uint32_t stream, unsigned long long drop_row,
                                                 int S, int key0, int lane) {
    slots[lane] = attn_dropout_block(seed, stream, (drop_row + (unsigned long long)(lane & 15) * S + key0 + (lane >> 4) * 32) >> 5);
}
// keep words of the packed pairs of rows r (k[j][0]) and r + 8 (k[j][1]) in column block j, from the warp's slots
__device__ __forceinline__ void warp_drop_words(const uint4* slots, uint32_t k2, int lane, uint32_t (&k)[8][2]) {
    const int r = lane >> 2;
#pragma unroll
    for (int g = 0; g < 2; ++g) {
        const uint4 ra = slots[g * 16 + r], rb = slots[g * 16 + r + 8];
#pragma unroll
        for (int w = 0; w < 4; ++w) {                             // column block j = 4g + w holds pair word 4w + lane % 4
            k[4 * g + w][0] = attn_dropout_word(ra, 4 * w + (lane & 3), k2);
            k[4 * g + w][1] = attn_dropout_word(rb, 4 * w + (lane & 3), k2);
        }
    }
}
// bf16 rows [r0, r0+16) x 64 columns of a fragment accumulator -> dqkv column block `col`; column sums of the stored values -> dbias.
// VARLEN: rows of packed sequence `sr`, only those below its length are stored and summed.
template <bool VARLEN>
__device__ __forceinline__ void store_rows_bf16(const AttnParams& p, const float (&acc)[8][4], float mul, int b, const SeqRows& sr,
                                                int s_row0, int col, int lane) {
    const int r = lane >> 2, c = 2 * (lane & 3);
    bf16* o0 = p.dqkv + (VARLEN ? sr.row0 + s_row0 + r : tok_row(p, b, s_row0 + r)) * (3LL * p.H) + col;
    bf16* o1 = p.dqkv + (VARLEN ? sr.row0 + s_row0 + r + 8 : tok_row(p, b, s_row0 + r + 8)) * (3LL * p.H) + col;
    const bool in0 = !VARLEN || s_row0 + r < sr.len, in1 = !VARLEN || s_row0 + r + 8 < sr.len;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const uint32_t u0 = pack_bf16(acc[j][0] * mul, acc[j][1] * mul), u1 = pack_bf16(acc[j][2] * mul, acc[j][3] * mul);
        if (in0) *reinterpret_cast<uint32_t*>(o0 + j * 8 + c) = u0;
        if (in1) *reinterpret_cast<uint32_t*>(o1 + j * 8 + c) = u1;
        if (p.dbias != nullptr) {
            const float2 f0 = in0 ? unpack_bf16(u0) : make_float2(0.f, 0.f), f1 = in1 ? unpack_bf16(u1) : make_float2(0.f, 0.f);
            float s0 = f0.x + f1.x, s1 = f0.y + f1.y;
#pragma unroll
            for (int o = 4; o < 32; o <<= 1) { s0 += __shfl_xor_sync(0xffffffffu, s0, o); s1 += __shfl_xor_sync(0xffffffffu, s1, o); }
            if (lane < 4) { atomicAdd(p.dbias + col + j * 8 + c, s0); atomicAdd(p.dbias + col + j * 8 + c + 1, s1); }
        }
    }
}
// dynamic shared memory rounded up to the 1024-byte alignment of the swizzled tiles
__device__ __forceinline__ uint8_t* smem_1k(uint8_t* smem) {
    return smem + (((smem_u32(smem) + 1023u) & ~1023u) - smem_u32(smem));
}

// =================================================================================================
// forward
// =================================================================================================
constexpr int FWD_WARPS = 8, FWD_THREADS = FWD_WARPS * 32, FWD_TQ = FWD_WARPS * 16;
constexpr int FWD_SMEM_BYTES = 1024 /*alignment*/ + 2 * TILE64_BYTES /*Q*/ + 4 * TILE64_BYTES /*K, V x 2*/ + 512 * 4 /*mask*/
                             + FWD_WARPS * 512 /*Philox blocks*/;

__global__ void __launch_bounds__(FWD_THREADS, 2)
attn_fwd_kernel(const AttnParams p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_1k(smem_raw);
    const int S = p.S, nkt = S / KT;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int qt = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
    const uint32_t sQ = smem_u32(smem), sK = sQ + 2 * TILE64_BYTES, sV = sK + 2 * TILE64_BYTES;
    float* sMask = reinterpret_cast<float*>(smem + 6 * TILE64_BYTES);      // additive mask of the key row, times log2(e)
    uint4* sRng = reinterpret_cast<uint4*>(smem + 6 * TILE64_BYTES + 512 * 4) + warp * 32;
    const long long ld = 3LL * p.H;

    load_tile<FWD_TQ, FWD_THREADS>(sQ, p.qkv, ld, h * HD, p, b, qt * FWD_TQ);
    load_tile<KT, FWD_THREADS>(sK, p.qkv, ld, p.H + h * HD, p, b, 0);
    load_tile<KT, FWD_THREADS>(sV, p.qkv, ld, 2 * p.H + h * HD, p, b, 0);
    cp_async_commit();
    for (int i = threadIdx.x; i < S; i += FWD_THREADS) sMask[i] = p.mask ? p.mask[(long long)b * S + i] * LOG2E : 0.f;

    const int r = lane >> 2, c = 2 * (lane & 3);
    const int q0 = qt * FWD_TQ + warp * 16 + r;                  // query rows q0 and q0 + 8 of this thread
    const uint32_t sQw = sQ + (warp >> 2) * TILE64_BYTES;        // the 64 query rows of this warpgroup
    const unsigned long long seed = effective_seed(p.seed, p.seed_dev);
    const unsigned long long drop_row = ((unsigned long long)(b * p.A + h) * S + qt * FWD_TQ + warp * 16) * (unsigned long long)S;
    float o[8][4];
#pragma unroll
    for (int j = 0; j < 8; ++j) o[j][0] = o[j][1] = o[j][2] = o[j][3] = 0.f;
    float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;

    for (int kt = 0; kt < nkt; ++kt) {
        const int buf = kt & 1;
        if (kt + 1 < nkt) {
            load_tile<KT, FWD_THREADS>(sK + (buf ^ 1) * TILE64_BYTES, p.qkv, ld, p.H + h * HD, p, b, (kt + 1) * KT);
            load_tile<KT, FWD_THREADS>(sV + (buf ^ 1) * TILE64_BYTES, p.qkv, ld, 2 * p.H + h * HD, p, b, (kt + 1) * KT);
        }
        cp_async_commit();
        tiles_ready<1>();
        float s[8][4];
        wgmma_fence();
        wg_abt(s, sQw, sK + buf * TILE64_BYTES);                 // S = Q K^T, in flight during the Philox blocks
        wgmma_commit();
        if (p.drop_on != 0u) warp_drop_blocks(sRng, seed, p.drop_stream, drop_row, S, kt * KT, lane);
        __syncwarp();
        wgmma_wait<0>();
        fence_regs(s);
        // ---- scale + mask (log2 domain), row maxima over the quad
        float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const float2 mk = *reinterpret_cast<const float2*>(sMask + kt * KT + j * 8 + c);
            s[j][0] = fmaf(s[j][0], p.scale_log2, mk.x); s[j][1] = fmaf(s[j][1], p.scale_log2, mk.y);
            s[j][2] = fmaf(s[j][2], p.scale_log2, mk.x); s[j][3] = fmaf(s[j][3], p.scale_log2, mk.y);
            mx0 = fmaxf(mx0, fmaxf(s[j][0], s[j][1])); mx1 = fmaxf(mx1, fmaxf(s[j][2], s[j][3]));
        }
#pragma unroll
        for (int off = 1; off < 4; off <<= 1) {
            mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, off)); mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, off));
        }
        const float mn0 = fmaxf(m0, mx0), mn1 = fmaxf(m1, mx1);
        const float al0 = ex2(m0 - mn0), al1 = ex2(m1 - mn1);          // 0 on the first tile (m = -inf)
        m0 = mn0; m1 = mn1;
        l0 *= al0; l1 *= al1;
#pragma unroll
        for (int j = 0; j < 8; ++j) { o[j][0] *= al0; o[j][1] *= al0; o[j][2] *= al1; o[j][3] *= al1; }
        // ---- p = exp2(s - m), row sums before dropout, P~ = keep-mask AND p (the 1/(1-p) scale is applied once, at the end)
        // P goes to the tensor core as bf16 hi + lo parts (two MMAs): O then carries P to ~16 significant bits, in step with the fp32
        // row sum l that normalises it -- a bf16 P alone leaves a per-element rounding of 2^-9 in O that l does not see.
        uint32_t pr[8][2], pl[8][2];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const float e0 = ex2(s[j][0] - mn0), e1 = ex2(s[j][1] - mn0), e2 = ex2(s[j][2] - mn1), e3 = ex2(s[j][3] - mn1);
            l0 += e0 + e1; l1 += e2 + e3;
            pr[j][0] = pack_bf16(e0, e1); pr[j][1] = pack_bf16(e2, e3);
            const float2 h0 = unpack_bf16(pr[j][0]), h1 = unpack_bf16(pr[j][1]);
            pl[j][0] = pack_bf16(e0 - h0.x, e1 - h0.y); pl[j][1] = pack_bf16(e2 - h1.x, e3 - h1.y);
        }
        if (p.drop_on != 0u) {
            uint32_t km[8][2];
            warp_drop_words(sRng, p.drop_k2, lane, km);
#pragma unroll
            for (int j = 0; j < 8; ++j) { pr[j][0] &= km[j][0]; pl[j][0] &= km[j][0]; pr[j][1] &= km[j][1]; pl[j][1] &= km[j][1]; }
        }
        fence_regs(o);
        wgmma_fence();
        wg_pt(o, pr, sV + buf * TILE64_BYTES);
        wg_pt(o, pl, sV + buf * TILE64_BYTES);
        wgmma_commit();
        wgmma_wait<0>();
        fence_regs(o); fence_regs(pr); fence_regs(pl);
        __syncthreads();                                                  // buffer `buf` is refilled at the next iteration
    }
    // ---- epilogue: O * (1/(1-p)) / l -> ctx, lse
#pragma unroll
    for (int off = 1; off < 4; off <<= 1) { l0 += __shfl_xor_sync(0xffffffffu, l0, off); l1 += __shfl_xor_sync(0xffffffffu, l1, off); }
    const float i0 = p.drop_scale / l0, i1 = p.drop_scale / l1;
    bf16* c0 = p.ctx + tok_row(p, b, q0) * p.H + h * HD;
    bf16* c1 = p.ctx + tok_row(p, b, q0 + 8) * p.H + h * HD;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        *reinterpret_cast<uint32_t*>(c0 + j * 8 + c) = pack_bf16(o[j][0] * i0, o[j][1] * i0);
        *reinterpret_cast<uint32_t*>(c1 + j * 8 + c) = pack_bf16(o[j][2] * i1, o[j][3] * i1);
    }
    if ((lane & 3) == 0) {
        float* lse = p.lse_out + ((long long)b * p.A + h) * S;
        lse[q0] = (m0 + log2f(l0)) * LN2;
        lse[q0 + 8] = (m1 + log2f(l1)) * LN2;
    }
}

// =================================================================================================
// variable-length forward: packed tokens, no mask.  TRAIN = false (inference): no dropout, no lse.  TRAIN = true: attn_fwd_kernel's
// dropout, keyed by the in-sequence (query, key) with stride drop_stride, and lse [A, T].
// =================================================================================================
struct VarlenParams {
    const bf16* qkv;           // [T, 3H], sequence b at rows cu_seqlens[b] .. cu_seqlens[b+1]
    const int* cu_seqlens;     // [B+1]
    bf16* ctx;                 // [T, H]
    int max_seqlen, H;
    float scale_log2;
    // TRAIN only
    float* lse_out;            // [A, T]: lse of (head h, token row t) at h*T + t
    int T, A, drop_stride;
    uint32_t drop_k2, drop_on; float drop_scale; uint32_t drop_stream; unsigned long long seed; const unsigned long long* seed_dev;
};
constexpr int FWD_VARLEN_SMEM_BYTES = 1024 /*alignment*/ + 2 * TILE64_BYTES /*Q*/ + 4 * TILE64_BYTES /*K, V x 2*/;
constexpr int FWD_VARLEN_TRAIN_SMEM_BYTES = FWD_VARLEN_SMEM_BYTES + FWD_WARPS * 512 /*Philox blocks*/;

// The tile body is attn_fwd_kernel's with the mask taken out.  A valid score goes through the same operations as there (fmaf with a
// zero addend; the padded kernel's extra terms for masked keys are exact zeros), so a row of a sequence gets the bits the padded
// kernel gives it under a -10000 mask of its padding -- with dropout too, when drop_stride = S.  Launched with FWD_THREADS threads; the
// register cap (instead of __launch_bounds__(FWD_THREADS, 2), which lets ptxas take 127) keeps the inference instance at
// attn_fwd_kernel's budget with no spills, and the training instance within 2 CTAs per SM.
template <bool TRAIN>
__global__ void __maxnreg__(TRAIN ? 128 : 120)
attn_fwd_varlen_kernel(const VarlenParams p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_1k(smem_raw);
    const int qt = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
    const long long row0 = p.cu_seqlens[b];
    const int len = max(0, min(p.cu_seqlens[b + 1] - (int)row0, p.max_seqlen));
    if (qt * FWD_TQ >= len) return;                              // CTA-uniform
    const int nkt = (len + KT - 1) / KT;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t sQ = smem_u32(smem), sK = sQ + 2 * TILE64_BYTES, sV = sK + 2 * TILE64_BYTES;
    const long long ld = 3LL * p.H;

    load_tile_varlen<FWD_TQ, FWD_THREADS>(sQ, p.qkv, ld, h * HD, row0, len, qt * FWD_TQ);
    load_tile_varlen<KT, FWD_THREADS>(sK, p.qkv, ld, p.H + h * HD, row0, len, 0);
    load_tile_varlen<KT, FWD_THREADS>(sV, p.qkv, ld, 2 * p.H + h * HD, row0, len, 0);
    cp_async_commit();

    const int r = lane >> 2, c = 2 * (lane & 3);
    const int q0 = qt * FWD_TQ + warp * 16 + r;                  // query rows q0 and q0 + 8 of this thread
    const uint32_t sQw = sQ + (warp >> 2) * TILE64_BYTES;
    uint4* sRng = nullptr;
    unsigned long long seed = 0, drop_row = 0;
    if constexpr (TRAIN) {
        sRng = reinterpret_cast<uint4*>(smem + 6 * TILE64_BYTES) + warp * 32;
        seed = effective_seed(p.seed, p.seed_dev);
        drop_row = ((unsigned long long)(b * p.A + h) * p.drop_stride + qt * FWD_TQ + warp * 16) * (unsigned long long)p.drop_stride;
    }
    float o[8][4];
#pragma unroll
    for (int j = 0; j < 8; ++j) o[j][0] = o[j][1] = o[j][2] = o[j][3] = 0.f;
    float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;

    for (int kt = 0; kt < nkt; ++kt) {
        const int buf = kt & 1;
        if (kt + 1 < nkt) {
            load_tile_varlen<KT, FWD_THREADS>(sK + (buf ^ 1) * TILE64_BYTES, p.qkv, ld, p.H + h * HD, row0, len, (kt + 1) * KT);
            load_tile_varlen<KT, FWD_THREADS>(sV + (buf ^ 1) * TILE64_BYTES, p.qkv, ld, 2 * p.H + h * HD, row0, len, (kt + 1) * KT);
        }
        cp_async_commit();
        tiles_ready<1>();
        float s[8][4];
        wgmma_fence();
        wg_abt(s, sQw, sK + buf * TILE64_BYTES);                 // S = Q K^T, in flight during the Philox blocks
        wgmma_commit();
        if constexpr (TRAIN) {
            if (p.drop_on != 0u) warp_drop_blocks(sRng, seed, p.drop_stream, drop_row, p.drop_stride, kt * KT, lane);
            __syncwarp();
        }
        wgmma_wait<0>();
        fence_regs(s);
        // ---- scale (log2 domain); keys at or past len (last tile only) -> -inf; row maxima over the quad
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            s[j][0] = fmaf(s[j][0], p.scale_log2, 0.f); s[j][1] = fmaf(s[j][1], p.scale_log2, 0.f);
            s[j][2] = fmaf(s[j][2], p.scale_log2, 0.f); s[j][3] = fmaf(s[j][3], p.scale_log2, 0.f);
        }
        if ((kt + 1) * KT > len) {
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const int key = kt * KT + j * 8 + c;
                if (key >= len) { s[j][0] = -INFINITY; s[j][2] = -INFINITY; }
                if (key + 1 >= len) { s[j][1] = -INFINITY; s[j][3] = -INFINITY; }
            }
        }
        float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
        for (int j = 0; j < 8; ++j) { mx0 = fmaxf(mx0, fmaxf(s[j][0], s[j][1])); mx1 = fmaxf(mx1, fmaxf(s[j][2], s[j][3])); }
#pragma unroll
        for (int off = 1; off < 4; off <<= 1) {
            mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, off)); mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, off));
        }
        const float mn0 = fmaxf(m0, mx0), mn1 = fmaxf(m1, mx1);    // finite: every tile holds key kt*64 < len
        const float al0 = ex2(m0 - mn0), al1 = ex2(m1 - mn1);
        m0 = mn0; m1 = mn1;
        l0 *= al0; l1 *= al1;
#pragma unroll
        for (int j = 0; j < 8; ++j) { o[j][0] *= al0; o[j][1] *= al0; o[j][2] *= al1; o[j][3] *= al1; }
        uint32_t pr[8][2], pl[8][2];                                        // P as bf16 hi + lo parts, as in attn_fwd_kernel
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const float e0 = ex2(s[j][0] - mn0), e1 = ex2(s[j][1] - mn0), e2 = ex2(s[j][2] - mn1), e3 = ex2(s[j][3] - mn1);
            l0 += e0 + e1; l1 += e2 + e3;
            pr[j][0] = pack_bf16(e0, e1); pr[j][1] = pack_bf16(e2, e3);
            const float2 h0 = unpack_bf16(pr[j][0]), h1 = unpack_bf16(pr[j][1]);
            pl[j][0] = pack_bf16(e0 - h0.x, e1 - h0.y); pl[j][1] = pack_bf16(e2 - h1.x, e3 - h1.y);
        }
        if constexpr (TRAIN) {
            if (p.drop_on != 0u) {                                          // P~ = keep-mask AND p, as in attn_fwd_kernel
                uint32_t km[8][2];
                warp_drop_words(sRng, p.drop_k2, lane, km);
#pragma unroll
                for (int j = 0; j < 8; ++j) { pr[j][0] &= km[j][0]; pl[j][0] &= km[j][0]; pr[j][1] &= km[j][1]; pl[j][1] &= km[j][1]; }
            }
        }
        fence_regs(o);
        wgmma_fence();
        wg_pt(o, pr, sV + buf * TILE64_BYTES);
        wg_pt(o, pl, sV + buf * TILE64_BYTES);
        wgmma_commit();
        wgmma_wait<0>();
        fence_regs(o); fence_regs(pr); fence_regs(pl);
        __syncthreads();                                                  // buffer `buf` is refilled at the next iteration
    }
    // ---- epilogue: O (* 1/(1-p)) / l -> ctx, rows below len only; lse (TRAIN)
#pragma unroll
    for (int off = 1; off < 4; off <<= 1) { l0 += __shfl_xor_sync(0xffffffffu, l0, off); l1 += __shfl_xor_sync(0xffffffffu, l1, off); }
    float i0, i1;
    if constexpr (TRAIN) { i0 = p.drop_scale / l0; i1 = p.drop_scale / l1; }
    else { i0 = 1.0f / l0; i1 = 1.0f / l1; }
    bf16* c0 = p.ctx + (row0 + q0) * p.H + h * HD;
    bf16* c1 = c0 + 8LL * p.H;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        if (q0 < len) *reinterpret_cast<uint32_t*>(c0 + j * 8 + c) = pack_bf16(o[j][0] * i0, o[j][1] * i0);
        if (q0 + 8 < len) *reinterpret_cast<uint32_t*>(c1 + j * 8 + c) = pack_bf16(o[j][2] * i1, o[j][3] * i1);
    }
    if constexpr (TRAIN) {
        if ((lane & 3) == 0) {
            float* lse = p.lse_out + (long long)h * p.T + row0;
            if (q0 < len) lse[q0] = (m0 + log2f(l0)) * LN2;
            if (q0 + 8 < len) lse[q0 + 8] = (m1 + log2f(l1)) * LN2;
        }
    }
}

// =================================================================================================
// backward
// =================================================================================================
constexpr int BWD_THREADS = 128;       // one warpgroup
// dK/dV keep words of one query tile: word i (0..15) of the Philox block of (query ql, key group g) at [(g*16 + i) * KEEP_LD + ql];
// the padding makes both the producer's row writes and the consumers' (ql, ql+1) pair reads free of bank conflicts
constexpr int KEEP_LD = 72;
constexpr int KEEP_BYTES = 32 * KEEP_LD * 4;
constexpr int BWD_DKV_SMEM_BYTES = 1024 + 6 * TILE64_BYTES + 2 * 512 * 4 /*-lse, -delta*/ + 2 * KEEP_BYTES;
constexpr int BWD_DQ_SMEM_BYTES = 1024 + 6 * TILE64_BYTES + 512 * 4 /*mask*/ + 4 * 512 /*Philox blocks*/;

// delta[b,h,s] = sum_d dO[t, h*64+d] * O[t, h*64+d].  Eight lanes share one (token, head) row: consecutive lanes read consecutive
// 16-byte units, so a warp instruction covers 4 whole 128-byte lines.
__global__ void attn_delta_kernel(const bf16* __restrict__ dctx, const bf16* __restrict__ ctx, float* __restrict__ delta,
                                  int B, int S, int A, int seq_first) {
    const long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long idx = gid >> 3;                                            // token * A + h
    const int unit = (int)(gid & 7);
    const long long total = (long long)B * S * A;
    float acc = 0.f;
    if (idx < total) {
        const uint4 ua = ld_global_nc_v4(dctx + idx * HD + unit * 8), uc = ld_global_nc_v4(ctx + idx * HD + unit * 8);
        float2 x, y;
        x = unpack_bf16(ua.x); y = unpack_bf16(uc.x); acc += x.x * y.x + x.y * y.y;
        x = unpack_bf16(ua.y); y = unpack_bf16(uc.y); acc += x.x * y.x + x.y * y.y;
        x = unpack_bf16(ua.z); y = unpack_bf16(uc.z); acc += x.x * y.x + x.y * y.y;
        x = unpack_bf16(ua.w); y = unpack_bf16(uc.w); acc += x.x * y.x + x.y * y.y;
    }
    acc += __shfl_xor_sync(0xffffffffu, acc, 1);
    acc += __shfl_xor_sync(0xffffffffu, acc, 2);
    acc += __shfl_xor_sync(0xffffffffu, acc, 4);
    if (idx < total && unit == 0) {
        const long long tok = idx / A; const int h = (int)(idx - tok * A);
        const int b = seq_first ? (int)(tok % B) : (int)(tok / S);
        const int s_ = seq_first ? (int)(tok / B) : (int)(tok - (long long)b * S);
        delta[((long long)b * A + h) * S + s_] = acc;
    }
}

// the 64 queries x 2 key groups of query tile qt against key tile kt: thread t computes the Philox block of (query t % 64, group
// t / 64) and all 16 of its pair words.  The keying stride is S, or drop_stride for packed sequences.
template <bool VARLEN>
__device__ __forceinline__ void dkv_keep_words(uint32_t* keep, const AttnParams& p, unsigned long long seed, long long bh, int kt, int qt) {
    const int ql = threadIdx.x & 63, g = threadIdx.x >> 6;
    const int stride = VARLEN ? p.drop_stride : p.S;
    const unsigned long long row = (unsigned long long)(bh * stride + qt * KT + ql) * (unsigned long long)stride;
    const uint4 blk = attn_dropout_block(seed, p.drop_stream, (row + kt * KT + g * 32) >> 5);
#pragma unroll
    for (int i = 0; i < 16; ++i) keep[(g * 16 + i) * KEEP_LD + ql] = attn_dropout_word(blk, i, p.drop_k2);
}

// dK, dV of one 64-key tile.  Thread layout of the transposed score tile: key rows kr, kr + 8 (kr = tile + warp*16 + lane/4),
// query columns 8j + 2(lane%4) + {0,1} of the current query tile.
//   P   = exp2(S * scale*log2e + mask*log2e - lse*log2e)          (bf16, as in forward)
//   P~  = keep-mask AND P
//   dS  = [ P~ * dP / (1-p) - P * delta ] * scale
//   dV += P~^T dO (times 1/(1-p) at the end),  dK += dS^T Q
// VARLEN: packed sequence b; the CTA walks its ceil(len/64) query tiles.  Query columns q >= len get -lse*log2e = -inf, so P and P~
// there are exactly ex2(-inf) = 0 whatever the (zero-filled) operands hold, and -delta*scale = 0; no lse or delta past len is read.
template <bool VARLEN>
__global__ void __launch_bounds__(BWD_THREADS)
attn_bwd_dkv_kernel(const AttnParams p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_1k(smem_raw);
    const SeqRows sr = VARLEN ? seq_rows(p.cu_seqlens, blockIdx.z, p.max_seqlen) : SeqRows{0, 0};
    if (VARLEN && (int)blockIdx.x * KT >= sr.len) return;       // CTA-uniform
    const int S = VARLEN ? (sr.len + KT - 1) / KT * KT : p.S, nqt = S / KT;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int kt = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
    const uint32_t sK = smem_u32(smem), sV = sK + TILE64_BYTES, sQ = sV + TILE64_BYTES, sdO = sQ + 2 * TILE64_BYTES;
    float* sLse = reinterpret_cast<float*>(smem + 6 * TILE64_BYTES);          // [S] -lse*log2e
    float* sNd = sLse + 512;                                                   // [S] -delta*scale
    uint32_t* sKeep = reinterpret_cast<uint32_t*>(sNd + 512);                  // 2 x [32 x KEEP_LD] keep words
    const long long ld = 3LL * p.H;
    const long long bh = (long long)b * p.A + h;

    load_rows<VARLEN, KT, BWD_THREADS>(sK, p.qkv, ld, p.H + h * HD, p, b, sr, kt * KT);
    load_rows<VARLEN, KT, BWD_THREADS>(sV, p.qkv, ld, 2 * p.H + h * HD, p, b, sr, kt * KT);
    load_rows<VARLEN, KT, BWD_THREADS>(sQ, p.qkv, ld, h * HD, p, b, sr, 0);
    load_rows<VARLEN, KT, BWD_THREADS>(sdO, p.dctx, p.H, h * HD, p, b, sr, 0);
    cp_async_commit();
    if constexpr (VARLEN) {
        const float* lse = p.lse + (long long)h * p.T + sr.row0;
        const float* delta = p.delta + (long long)h * p.T + sr.row0;
        for (int i = threadIdx.x; i < S; i += BWD_THREADS) {
            const bool in = i < sr.len;
            sLse[i] = in ? -lse[i] * LOG2E : -INFINITY;
            sNd[i] = in ? -delta[i] * p.scale : 0.f;
        }
    } else {
        for (int i = threadIdx.x; i < S; i += BWD_THREADS) { sLse[i] = -p.lse[bh * S + i] * LOG2E; sNd[i] = -p.delta[bh * S + i] * p.scale; }
    }
    const unsigned long long seed = effective_seed(p.seed, p.seed_dev);
    if (p.drop_on != 0u) dkv_keep_words<VARLEN>(sKeep, p, seed, bh, kt, 0);

    const int r = lane >> 2, c = 2 * (lane & 3);
    const int kr = kt * KT + warp * 16 + r;                      // key rows kr and kr + 8 of this thread
    const float mk0 = (!VARLEN && p.mask) ? p.mask[(long long)b * S + kr] * LOG2E : 0.f;
    const float mk1 = (!VARLEN && p.mask) ? p.mask[(long long)b * S + kr + 8] * LOG2E : 0.f;
    // keys kr and kr + 8 are halves (r & 1) of pair words i and i + 4 of key group warp / 2, for every query
    const int keep_row = (warp >> 1) * 16 + (warp & 1) * 8 + (r >> 1);
    const uint32_t half_sel = (r & 1) ? 0x7632u : 0x5410u;
    const float c1 = p.drop_scale * p.scale;
    float dk[8][4], dv[8][4];
#pragma unroll
    for (int j = 0; j < 8; ++j) { dk[j][0] = dk[j][1] = dk[j][2] = dk[j][3] = 0.f; dv[j][0] = dv[j][1] = dv[j][2] = dv[j][3] = 0.f; }

    for (int qt = 0; qt < nqt; ++qt) {
        const int buf = qt & 1;
        if (qt + 1 < nqt) {
            load_rows<VARLEN, KT, BWD_THREADS>(sQ + (buf ^ 1) * TILE64_BYTES, p.qkv, ld, h * HD, p, b, sr, (qt + 1) * KT);
            load_rows<VARLEN, KT, BWD_THREADS>(sdO + (buf ^ 1) * TILE64_BYTES, p.dctx, p.H, h * HD, p, b, sr, (qt + 1) * KT);
        }
        cp_async_commit();
        tiles_ready<1>();                                        // also publishes the keep words of this query tile
        const uint32_t tQ = sQ + buf * TILE64_BYTES, tdO = sdO + buf * TILE64_BYTES;
        float st[8][4], dpt[8][4];
        wgmma_fence();
        wg_abt(st, sK, tQ);                                      // S^T  = K Q^T
        wg_abt(dpt, sV, tdO);                                    // dP^T = V dO^T
        wgmma_commit();
        // while the MMAs run: the keep words of the next query tile (read after the next iteration's barrier)
        if (p.drop_on != 0u && qt + 1 < nqt) dkv_keep_words<VARLEN>(sKeep + ((qt + 1) & 1) * (32 * KEEP_LD), p, seed, bh, kt, qt + 1);
        wgmma_wait<0>();
        fence_regs(st); fence_regs(dpt);
        const uint32_t* keep = sKeep + buf * (32 * KEEP_LD) + keep_row * KEEP_LD;
        uint32_t pm[8][2], ds[8][2];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int q = qt * KT + j * 8 + c;                   // query columns q, q + 1
            const float2 nl = *reinterpret_cast<const float2*>(sLse + q);
            const float2 nd = *reinterpret_cast<const float2*>(sNd + q);
            const uint32_t p0 = pack_bf16(ex2(fmaf(st[j][0], p.scale_log2, mk0) + nl.x), ex2(fmaf(st[j][1], p.scale_log2, mk0) + nl.y));
            const uint32_t p1 = pack_bf16(ex2(fmaf(st[j][2], p.scale_log2, mk1) + nl.x), ex2(fmaf(st[j][3], p.scale_log2, mk1) + nl.y));
            uint32_t k0 = 0xFFFFFFFFu, k1 = 0xFFFFFFFFu;
            if (p.drop_on != 0u) {
                const uint2 wa = *reinterpret_cast<const uint2*>(keep + j * 8 + c);                 // word i of queries q, q + 1
                const uint2 wb = *reinterpret_cast<const uint2*>(keep + 4 * KEEP_LD + j * 8 + c);   // word i + 4
                k0 = prmt(wa.x, wa.y, half_sel);
                k1 = prmt(wb.x, wb.y, half_sel);
            }
            pm[j][0] = p0 & k0; pm[j][1] = p1 & k1;
            const float2 f0 = unpack_bf16(p0), f1 = unpack_bf16(p1), g0 = unpack_bf16(pm[j][0]), g1 = unpack_bf16(pm[j][1]);
            ds[j][0] = pack_bf16(fmaf(g0.x * dpt[j][0], c1, f0.x * nd.x), fmaf(g0.y * dpt[j][1], c1, f0.y * nd.y));
            ds[j][1] = pack_bf16(fmaf(g1.x * dpt[j][2], c1, f1.x * nd.x), fmaf(g1.y * dpt[j][3], c1, f1.y * nd.y));
        }
        fence_regs(dv); fence_regs(dk);
        wgmma_fence();
        wg_pt(dv, pm, tdO);                                      // dV += P~^T dO
        wg_pt(dk, ds, tQ);                                       // dK += dS^T Q
        wgmma_commit();
        wgmma_wait<0>();
        fence_regs(dv); fence_regs(dk); fence_regs(pm); fence_regs(ds);
        __syncthreads();
    }
    const int s_row0 = kt * KT + warp * 16;
    store_rows_bf16<VARLEN>(p, dk, 1.0f, b, sr, s_row0, p.H + h * HD, lane);
    store_rows_bf16<VARLEN>(p, dv, p.drop_scale, b, sr, s_row0, 2 * p.H + h * HD, lane);
}

// t - lse*log2e for a scaled, masked score t.  The padded dQ instance passes l = -lse*log2e, and ptxas contracts that add into
// fma(lse, -log2e, t); the packed instance passes l = lse and states the fma, so that both round once and P agrees bit for bit.
template <bool VARLEN>
__device__ __forceinline__ float minus_lse(float t, float l) {
    if constexpr (VARLEN) return fmaf(l, -LOG2E, t);
    else return t + l;
}

// dQ of one 64-query tile: rows q, q + 8 (q = tile + warp*16 + lane/4), key columns of the current key tile.  dQ += dS K.
// VARLEN: packed sequence b; the CTA walks its ceil(len/64) key tiles.  Key columns k >= len get an additive -inf mask, so P and P~
// there are exactly 0; the lse / delta of query rows q >= len (never stored) are not read.
template <bool VARLEN>
__global__ void __launch_bounds__(BWD_THREADS)
attn_bwd_dq_kernel(const AttnParams p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_1k(smem_raw);
    const SeqRows sr = VARLEN ? seq_rows(p.cu_seqlens, blockIdx.z, p.max_seqlen) : SeqRows{0, 0};
    if (VARLEN && (int)blockIdx.x * KT >= sr.len) return;       // CTA-uniform
    const int S = VARLEN ? (sr.len + KT - 1) / KT * KT : p.S, nkt = S / KT;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int qt = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
    const int stride = VARLEN ? p.drop_stride : S;
    const uint32_t sQ = smem_u32(smem), sdO = sQ + TILE64_BYTES, sK = sdO + TILE64_BYTES, sV = sK + 2 * TILE64_BYTES;
    float* sMask = reinterpret_cast<float*>(smem + 6 * TILE64_BYTES);
    uint4* sRng = reinterpret_cast<uint4*>(smem + 6 * TILE64_BYTES + 512 * 4) + warp * 32;
    const long long ld = 3LL * p.H;
    const long long bh = (long long)b * p.A + h;

    load_rows<VARLEN, KT, BWD_THREADS>(sQ, p.qkv, ld, h * HD, p, b, sr, qt * KT);
    load_rows<VARLEN, KT, BWD_THREADS>(sdO, p.dctx, p.H, h * HD, p, b, sr, qt * KT);
    load_rows<VARLEN, KT, BWD_THREADS>(sK, p.qkv, ld, p.H + h * HD, p, b, sr, 0);
    load_rows<VARLEN, KT, BWD_THREADS>(sV, p.qkv, ld, 2 * p.H + h * HD, p, b, sr, 0);
    cp_async_commit();
    if constexpr (VARLEN) {
        for (int i = threadIdx.x; i < S; i += BWD_THREADS) sMask[i] = i < sr.len ? 0.f : -INFINITY;
    } else {
        for (int i = threadIdx.x; i < S; i += BWD_THREADS) sMask[i] = p.mask ? p.mask[(long long)b * S + i] * LOG2E : 0.f;
    }

    const int r = lane >> 2, c = 2 * (lane & 3);
    const int q0 = qt * KT + warp * 16 + r;
    float nl0, nl1, nd0, nd1;
    if constexpr (VARLEN) {
        const float* lse = p.lse + (long long)h * p.T + sr.row0;
        const float* delta = p.delta + (long long)h * p.T + sr.row0;
        const bool in0 = q0 < sr.len, in1 = q0 + 8 < sr.len;
        nl0 = in0 ? lse[q0] : 0.f; nl1 = in1 ? lse[q0 + 8] : 0.f;                   // raw lse: see minus_lse
        nd0 = in0 ? -delta[q0] * p.scale : 0.f; nd1 = in1 ? -delta[q0 + 8] * p.scale : 0.f;
    } else {
        nl0 = -p.lse[bh * S + q0] * LOG2E; nl1 = -p.lse[bh * S + q0 + 8] * LOG2E;
        nd0 = -p.delta[bh * S + q0] * p.scale; nd1 = -p.delta[bh * S + q0 + 8] * p.scale;
    }
    const unsigned long long seed = effective_seed(p.seed, p.seed_dev);
    const unsigned long long drop_row = (unsigned long long)(bh * stride + qt * KT + warp * 16) * (unsigned long long)stride;
    const float c1 = p.drop_scale * p.scale;
    float dq[8][4];
#pragma unroll
    for (int j = 0; j < 8; ++j) dq[j][0] = dq[j][1] = dq[j][2] = dq[j][3] = 0.f;

    for (int kt = 0; kt < nkt; ++kt) {
        const int buf = kt & 1;
        if (kt + 1 < nkt) {
            load_rows<VARLEN, KT, BWD_THREADS>(sK + (buf ^ 1) * TILE64_BYTES, p.qkv, ld, p.H + h * HD, p, b, sr, (kt + 1) * KT);
            load_rows<VARLEN, KT, BWD_THREADS>(sV + (buf ^ 1) * TILE64_BYTES, p.qkv, ld, 2 * p.H + h * HD, p, b, sr, (kt + 1) * KT);
        }
        cp_async_commit();
        tiles_ready<1>();
        const uint32_t tK = sK + buf * TILE64_BYTES, tV = sV + buf * TILE64_BYTES;
        float s[8][4], dp[8][4];
        wgmma_fence();
        wg_abt(s, sQ, tK);                                       // S  = Q K^T
        wg_abt(dp, sdO, tV);                                     // dP = dO V^T
        wgmma_commit();
        if (p.drop_on != 0u) warp_drop_blocks(sRng, seed, p.drop_stream, drop_row, stride, kt * KT, lane);
        __syncwarp();
        uint32_t km[8][2];
#pragma unroll
        for (int j = 0; j < 8; ++j) km[j][0] = km[j][1] = 0xFFFFFFFFu;
        if (p.drop_on != 0u) warp_drop_words(sRng, p.drop_k2, lane, km);
        wgmma_wait<0>();
        fence_regs(s); fence_regs(dp);
        uint32_t ds[8][2];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const float2 mk = *reinterpret_cast<const float2*>(sMask + kt * KT + j * 8 + c);
            const uint32_t p0 = pack_bf16(ex2(minus_lse<VARLEN>(fmaf(s[j][0], p.scale_log2, mk.x), nl0)),
                                          ex2(minus_lse<VARLEN>(fmaf(s[j][1], p.scale_log2, mk.y), nl0)));
            const uint32_t p1 = pack_bf16(ex2(minus_lse<VARLEN>(fmaf(s[j][2], p.scale_log2, mk.x), nl1)),
                                          ex2(minus_lse<VARLEN>(fmaf(s[j][3], p.scale_log2, mk.y), nl1)));
            const float2 f0 = unpack_bf16(p0), f1 = unpack_bf16(p1), g0 = unpack_bf16(p0 & km[j][0]), g1 = unpack_bf16(p1 & km[j][1]);
            ds[j][0] = pack_bf16(fmaf(g0.x * dp[j][0], c1, f0.x * nd0), fmaf(g0.y * dp[j][1], c1, f0.y * nd0));
            ds[j][1] = pack_bf16(fmaf(g1.x * dp[j][2], c1, f1.x * nd1), fmaf(g1.y * dp[j][3], c1, f1.y * nd1));
        }
        fence_regs(dq);
        wgmma_fence();
        wg_pt(dq, ds, tK);                                       // dQ += dS K
        wgmma_commit();
        wgmma_wait<0>();
        fence_regs(dq); fence_regs(ds);
        __syncthreads();
    }
    store_rows_bf16<VARLEN>(p, dq, 1.0f, b, sr, qt * KT + warp * 16, h * HD, lane);
}

}  // namespace dle

using namespace dle;

// dropout probability -> the kernels' parameters.  p is quantised to 1/32768 (common.cuh: attn_dropout_word); the rescale uses the
// quantised value so that E[P~] = P exactly.
static void attn_drop_params(float dropout_p, uint32_t* k2, uint32_t* on, float* scale) {
    const uint32_t t15 = dropout_p > 0.f ? dropout_thresh15(dropout_p) : 0u;
    *on = t15 != 0u ? 1u : 0u;
    *k2 = attn_dropout_k2(t15);
    *scale = t15 != 0u ? 1.0f / (1.0f - (float)t15 / 32768.0f) : 1.0f;
}
// cudaFuncAttributeMaxDynamicSharedMemorySize is a per-device attribute: remember which devices have it (per kernel)
struct SmemAttrCache { int bytes[64] = {0}; };
template <typename K>
static int ensure_smem_attr(K kern, SmemAttrCache& c, int bytes) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return DLE_ERR_CUDA;
    if (bytes > c.bytes[dev]) {
        if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes) != cudaSuccess) return DLE_ERR_CUDA;
        c.bytes[dev] = bytes;
    }
    return DLE_OK;
}

static int attn_check(int B, int S, int A) {
    if (B <= 0 || A <= 0 || S <= 0 || S % 128 != 0 || S > 512) return DLE_ERR_INVALID;
    return DLE_OK;
}
static void attn_common(AttnParams& p, const void* qkv, const float* mask, int B, int S, int A, int seq_first, float dropout_p,
                        uint64_t seed, const uint64_t* seed_dev, uint32_t dropout_stream) {
    p = AttnParams{};
    p.qkv = reinterpret_cast<const bf16*>(qkv); p.mask = mask;
    p.B = B; p.S = S; p.A = A; p.H = A * HD;
    p.tok_stride_s = seq_first ? B : 1; p.tok_stride_b = seq_first ? 1 : S;
    p.scale = 0.125f; p.scale_log2 = 0.125f * LOG2E;
    attn_drop_params(dropout_p, &p.drop_k2, &p.drop_on, &p.drop_scale);
    p.drop_stream = dropout_stream; p.seed = seed; p.seed_dev = reinterpret_cast<const unsigned long long*>(seed_dev);
}
static bool aligned16(const void* x) { return (reinterpret_cast<uintptr_t>(x) & 15) == 0; }

extern "C" int dle_attn_fwd(const void* qkv, const float* mask, void* ctx, float* lse, int32_t B, int32_t S, int32_t A,
                            int32_t seq_first, float dropout_p, uint64_t seed, const uint64_t* seed_dev, uint32_t dropout_stream, void* stream) {
    DLE_CHECK_ARG(qkv && ctx && lse && attn_check(B, S, A) == DLE_OK && dropout_p >= 0.f && dropout_p < 1.f);
    DLE_CHECK_ARG(aligned16(qkv) && aligned16(ctx));
    AttnParams p;
    attn_common(p, qkv, mask, B, S, A, seq_first, dropout_p, seed, seed_dev, dropout_stream);
    p.ctx = reinterpret_cast<bf16*>(ctx); p.lse_out = lse;
    static SmemAttrCache attr;
    int rc = ensure_smem_attr(attn_fwd_kernel, attr, FWD_SMEM_BYTES);
    if (rc != DLE_OK) return rc;
    attn_fwd_kernel<<<dim3(S / FWD_TQ, A, B), FWD_THREADS, FWD_SMEM_BYTES, reinterpret_cast<cudaStream_t>(stream)>>>(p);
    DLE_LAUNCH_CHECK();
    return DLE_OK;
}

extern "C" int dle_attn_fwd_varlen(const void* qkv, const int32_t* cu_seqlens, void* ctx, int32_t B, int32_t max_seqlen, int32_t A,
                                   void* stream) {
    DLE_CHECK_ARG(qkv && cu_seqlens && ctx && B > 0 && B <= 65535 && A > 0 && A <= 65535 && max_seqlen >= 1 && max_seqlen <= 512);
    DLE_CHECK_ARG(aligned16(qkv) && aligned16(ctx) && (reinterpret_cast<uintptr_t>(cu_seqlens) & 3) == 0);
    VarlenParams p{};
    p.qkv = reinterpret_cast<const bf16*>(qkv); p.cu_seqlens = cu_seqlens; p.ctx = reinterpret_cast<bf16*>(ctx);
    p.max_seqlen = max_seqlen; p.H = A * HD; p.scale_log2 = 0.125f * LOG2E;
    static SmemAttrCache attr;
    int rc = ensure_smem_attr(attn_fwd_varlen_kernel<false>, attr, FWD_VARLEN_SMEM_BYTES);
    if (rc != DLE_OK) return rc;
    attn_fwd_varlen_kernel<false><<<dim3((max_seqlen + FWD_TQ - 1) / FWD_TQ, A, B), FWD_THREADS, FWD_VARLEN_SMEM_BYTES,
                             reinterpret_cast<cudaStream_t>(stream)>>>(p);
    DLE_LAUNCH_CHECK();
    return DLE_OK;
}

extern "C" int dle_attn_bwd(const void* qkv, const float* mask, const void* ctx, const void* dctx, const float* lse, void* dqkv,
                            float* delta_ws, float* dbias_qkv, int32_t B, int32_t S, int32_t A, int32_t seq_first, float dropout_p, uint64_t seed,
                            const uint64_t* seed_dev, uint32_t dropout_stream, void* stream) {
    DLE_CHECK_ARG(qkv && ctx && dctx && lse && dqkv && delta_ws && attn_check(B, S, A) == DLE_OK && dropout_p >= 0.f && dropout_p < 1.f);
    DLE_CHECK_ARG(aligned16(qkv) && aligned16(ctx) && aligned16(dctx) && aligned16(dqkv));
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const long long total = (long long)B * S * A;
    attn_delta_kernel<<<(unsigned)((total * 8 + 255) / 256), 256, 0, st>>>(reinterpret_cast<const bf16*>(dctx), reinterpret_cast<const bf16*>(ctx), delta_ws, B, S, A, seq_first);
    DLE_LAUNCH_CHECK();
    AttnParams p;
    attn_common(p, qkv, mask, B, S, A, seq_first, dropout_p, seed, seed_dev, dropout_stream);
    p.dctx = reinterpret_cast<const bf16*>(dctx); p.lse = lse; p.delta = delta_ws; p.dbias = dbias_qkv; p.dqkv = reinterpret_cast<bf16*>(dqkv);
    static SmemAttrCache attr_kv, attr_q;
    int rc = ensure_smem_attr(attn_bwd_dkv_kernel<false>, attr_kv, BWD_DKV_SMEM_BYTES);
    if (rc != DLE_OK) return rc;
    rc = ensure_smem_attr(attn_bwd_dq_kernel<false>, attr_q, BWD_DQ_SMEM_BYTES);
    if (rc != DLE_OK) return rc;
    attn_bwd_dkv_kernel<false><<<dim3(S / KT, A, B), BWD_THREADS, BWD_DKV_SMEM_BYTES, st>>>(p);
    DLE_LAUNCH_CHECK();
    attn_bwd_dq_kernel<false><<<dim3(S / KT, A, B), BWD_THREADS, BWD_DQ_SMEM_BYTES, st>>>(p);
    DLE_LAUNCH_CHECK();
    return DLE_OK;
}

// shared argument checks of the packed training entry points
static bool varlen_train_args_ok(int T, int B, int max_seqlen, int A, int drop_stride, float dropout_p) {
    return T > 0 && B > 0 && B <= 65535 && A > 0 && A <= 65535 && max_seqlen >= 1 && max_seqlen <= 512 && drop_stride % 64 == 0 &&
           drop_stride >= max_seqlen && drop_stride <= 512 && dropout_p >= 0.f && dropout_p < 1.f;
}

extern "C" int dle_attn_fwd_varlen_train(const void* qkv, const int32_t* cu_seqlens, void* ctx, float* lse, int32_t T, int32_t B,
                                         int32_t max_seqlen, int32_t A, int32_t drop_stride, float dropout_p, uint64_t seed,
                                         const uint64_t* seed_dev, uint32_t dropout_stream, void* stream) {
    DLE_CHECK_ARG(qkv && cu_seqlens && ctx && lse && varlen_train_args_ok(T, B, max_seqlen, A, drop_stride, dropout_p));
    DLE_CHECK_ARG(aligned16(qkv) && aligned16(ctx) && (reinterpret_cast<uintptr_t>(cu_seqlens) & 3) == 0 &&
                  (reinterpret_cast<uintptr_t>(lse) & 3) == 0);
    VarlenParams p{};
    p.qkv = reinterpret_cast<const bf16*>(qkv); p.cu_seqlens = cu_seqlens; p.ctx = reinterpret_cast<bf16*>(ctx);
    p.max_seqlen = max_seqlen; p.H = A * HD; p.scale_log2 = 0.125f * LOG2E;
    p.lse_out = lse; p.T = T; p.A = A; p.drop_stride = drop_stride;
    attn_drop_params(dropout_p, &p.drop_k2, &p.drop_on, &p.drop_scale);
    p.drop_stream = dropout_stream; p.seed = seed; p.seed_dev = reinterpret_cast<const unsigned long long*>(seed_dev);
    static SmemAttrCache attr;
    int rc = ensure_smem_attr(attn_fwd_varlen_kernel<true>, attr, FWD_VARLEN_TRAIN_SMEM_BYTES);
    if (rc != DLE_OK) return rc;
    attn_fwd_varlen_kernel<true><<<dim3((max_seqlen + FWD_TQ - 1) / FWD_TQ, A, B), FWD_THREADS, FWD_VARLEN_TRAIN_SMEM_BYTES,
                                    reinterpret_cast<cudaStream_t>(stream)>>>(p);
    DLE_LAUNCH_CHECK();
    return DLE_OK;
}

extern "C" int dle_attn_bwd_varlen(const void* qkv, const int32_t* cu_seqlens, const void* ctx, const void* dctx, const float* lse,
                                   void* dqkv, float* delta_ws, float* dbias_qkv, int32_t T, int32_t B, int32_t max_seqlen, int32_t A,
                                   int32_t drop_stride, float dropout_p, uint64_t seed, const uint64_t* seed_dev, uint32_t dropout_stream,
                                   void* stream) {
    DLE_CHECK_ARG(qkv && cu_seqlens && ctx && dctx && lse && dqkv && delta_ws &&
                  varlen_train_args_ok(T, B, max_seqlen, A, drop_stride, dropout_p));
    DLE_CHECK_ARG(aligned16(qkv) && aligned16(ctx) && aligned16(dctx) && aligned16(dqkv) && (reinterpret_cast<uintptr_t>(cu_seqlens) & 3) == 0 &&
                  (reinterpret_cast<uintptr_t>(lse) & 3) == 0 && (reinterpret_cast<uintptr_t>(delta_ws) & 3) == 0 &&
                  (reinterpret_cast<uintptr_t>(dbias_qkv) & 3) == 0);
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    // delta [A, T]: the padded kernel's arithmetic over one "sequence" of all T rows
    const long long total = (long long)T * A;
    attn_delta_kernel<<<(unsigned)((total * 8 + 255) / 256), 256, 0, st>>>(reinterpret_cast<const bf16*>(dctx), reinterpret_cast<const bf16*>(ctx), delta_ws, 1, T, A, 0);
    DLE_LAUNCH_CHECK();
    AttnParams p;
    attn_common(p, qkv, nullptr, B, 0, A, 0, dropout_p, seed, seed_dev, dropout_stream);
    p.dctx = reinterpret_cast<const bf16*>(dctx); p.lse = lse; p.delta = delta_ws; p.dbias = dbias_qkv; p.dqkv = reinterpret_cast<bf16*>(dqkv);
    p.cu_seqlens = cu_seqlens; p.T = T; p.max_seqlen = max_seqlen; p.drop_stride = drop_stride;
    static SmemAttrCache attr_kv, attr_q;
    int rc = ensure_smem_attr(attn_bwd_dkv_kernel<true>, attr_kv, BWD_DKV_SMEM_BYTES);
    if (rc != DLE_OK) return rc;
    rc = ensure_smem_attr(attn_bwd_dq_kernel<true>, attr_q, BWD_DQ_SMEM_BYTES);
    if (rc != DLE_OK) return rc;
    const dim3 grid((max_seqlen + KT - 1) / KT, A, B);
    attn_bwd_dkv_kernel<true><<<grid, BWD_THREADS, BWD_DKV_SMEM_BYTES, st>>>(p);
    DLE_LAUNCH_CHECK();
    attn_bwd_dq_kernel<true><<<grid, BWD_THREADS, BWD_DQ_SMEM_BYTES, st>>>(p);
    DLE_LAUNCH_CHECK();
    return DLE_OK;
}
