// Fused multi-head self-attention for sm_90a (head dim 64, S in {128,256,384,512}), on the warp-level tensor-core MMA
// (mma.sync m16n8k16, bf16 in, fp32 accumulate) with operands fed from XOR-swizzled shared memory by ldmatrix and tiles
// streamed in by cp.async double buffering.
//
// Forward : one CTA per (batch, head, 128-query tile), 8 warps x 16 query rows.  Q stays in registers; K / V come in 64-key
//           tiles.  S = Q K^T, online softmax in registers, dropout (Philox, regenerated in backward), O += P V with P taken
//           straight from the S accumulators (as bf16 hi + lo parts).  The [B,A,S,S] score tensor the reference materialises 3x per layer never
//           exists in HBM.
// Backward: two kernels that recompute P from the saved log-sum-exp, so that every output is accumulated on chip by exactly
//           one CTA -- no atomics on dQ / dK / dV, deterministic:
//             dK / dV : one CTA per (batch, head, 64-key tile); the warps hold their 16 keys' K and V rows in registers and
//                       walk the query tiles, computing S^T = K Q^T and dP^T = V dO^T, then dV += P~^T dO, dK += dS^T Q.
//             dQ      : one CTA per (batch, head, 64-query tile); the warps hold Q and dO rows and walk the key tiles,
//                       computing S and dP again, then dQ += dS K.
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
// byte offset of 16-byte unit `ch` (8 bf16) of row r in a tile of 128-byte rows, XOR-swizzled by row % 8 so that both the
// cp.async row writes and the ldmatrix 8-row reads are free of bank conflicts
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
};

__device__ __forceinline__ long long tok_row(const AttnParams& p, int b, int s) {
    return (long long)b * p.tok_stride_b + (long long)s * p.tok_stride_s;
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
// A fragments (16 rows from r0, all 64 columns = 4 k-steps) of a swizzled tile
__device__ __forceinline__ void load_a_frags(uint32_t tile, int r0, int lane, uint32_t (&f)[4][4]) {
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) ldsm_x4(tile + sw(r0 + (lane & 15), 2 * kk + (lane >> 4)), f[kk][0], f[kk][1], f[kk][2], f[kk][3]);
}
// acc[16 x 64] = A[16 x 64] * T^T where tile T holds 64 rows (the n dimension) of 64 columns (the k dimension)
__device__ __forceinline__ void mma_abt(float (&acc)[8][4], const uint32_t (&a)[4][4], uint32_t tile, int lane) {
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f;
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
#pragma unroll
        for (int np = 0; np < 4; ++np) {
            uint32_t b0, b1, b2, b3;
            ldsm_x4(tile + sw(16 * np + (lane & 7) + ((lane >> 4) << 3), 2 * kk + ((lane >> 3) & 1)), b0, b1, b2, b3);
            mma_bf16_16816(acc[2 * np], a[kk], b0, b1);
            mma_bf16_16816(acc[2 * np + 1], a[kk], b2, b3);
        }
    }
}
// acc[16 x 64] += A[16 x 64] * T where A arrives as packed bf16 accumulator pairs (pr[j][0]: row r, pr[j][1]: row r + 8 of
// column tile j) and tile T holds 64 rows (the k dimension) of 64 columns (the n dimension)
__device__ __forceinline__ void mma_pt(float (&acc)[8][4], const uint32_t (&pr)[8][2], uint32_t tile, int lane) {
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
        const uint32_t a[4] = {pr[2 * kk][0], pr[2 * kk][1], pr[2 * kk + 1][0], pr[2 * kk + 1][1]};
#pragma unroll
        for (int np = 0; np < 4; ++np) {
            uint32_t b0, b1, b2, b3;
            ldsm_x4_trans(tile + sw(16 * kk + (lane & 7) + (((lane >> 3) & 1) << 3), 2 * np + (lane >> 4)), b0, b1, b2, b3);
            mma_bf16_16816(acc[2 * np], a, b0, b1);
            mma_bf16_16816(acc[2 * np + 1], a, b2, b3);
        }
    }
}
// 16-bit keep mask of one element: 0xFFFF (kept) or 0
__device__ __forceinline__ uint32_t keep_half(const uint4& r, int key, uint32_t k2) {
    const uint32_t w = attn_dropout_word(r, (key & 31) >> 1, k2);
    return (key & 1) ? (w >> 16) : (w & 0xFFFFu);
}
// bf16 rows [r0, r0+16) x 64 columns of a fragment accumulator -> dqkv column block `col`; column sums of the stored values -> dbias
__device__ __forceinline__ void store_rows_bf16(const AttnParams& p, const float (&acc)[8][4], float mul, int b, int s_row0, int col, int lane) {
    const int r = lane >> 2, c = 2 * (lane & 3);
    bf16* o0 = p.dqkv + tok_row(p, b, s_row0 + r) * (3LL * p.H) + col;
    bf16* o1 = p.dqkv + tok_row(p, b, s_row0 + r + 8) * (3LL * p.H) + col;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const uint32_t u0 = pack_bf16(acc[j][0] * mul, acc[j][1] * mul), u1 = pack_bf16(acc[j][2] * mul, acc[j][3] * mul);
        *reinterpret_cast<uint32_t*>(o0 + j * 8 + c) = u0;
        *reinterpret_cast<uint32_t*>(o1 + j * 8 + c) = u1;
        if (p.dbias != nullptr) {
            const float2 f0 = unpack_bf16(u0), f1 = unpack_bf16(u1);
            float s0 = f0.x + f1.x, s1 = f0.y + f1.y;
#pragma unroll
            for (int o = 4; o < 32; o <<= 1) { s0 += __shfl_xor_sync(0xffffffffu, s0, o); s1 += __shfl_xor_sync(0xffffffffu, s1, o); }
            if (lane < 4) { atomicAdd(p.dbias + col + j * 8 + c, s0); atomicAdd(p.dbias + col + j * 8 + c + 1, s1); }
        }
    }
}

// =================================================================================================
// forward
// =================================================================================================
constexpr int FWD_WARPS = 8, FWD_THREADS = FWD_WARPS * 32, FWD_TQ = FWD_WARPS * 16;
constexpr int FWD_SMEM_BYTES = 2 * TILE64_BYTES /*Q*/ + 4 * TILE64_BYTES /*K, V x 2*/ + 512 * 4 /*mask*/;

__global__ void __launch_bounds__(FWD_THREADS)
attn_fwd_kernel(const AttnParams p) {
    extern __shared__ __align__(128) uint8_t smem[];
    const int S = p.S, nkt = S / KT;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int qt = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
    const uint32_t sQ = smem_u32(smem), sK = sQ + 2 * TILE64_BYTES, sV = sK + 2 * TILE64_BYTES;
    float* sMask = reinterpret_cast<float*>(smem + 6 * TILE64_BYTES);      // additive mask of the key row, times log2(e)
    const long long ld = 3LL * p.H;

    load_tile<FWD_TQ, FWD_THREADS>(sQ, p.qkv, ld, h * HD, p, b, qt * FWD_TQ);
    load_tile<KT, FWD_THREADS>(sK, p.qkv, ld, p.H + h * HD, p, b, 0);
    load_tile<KT, FWD_THREADS>(sV, p.qkv, ld, 2 * p.H + h * HD, p, b, 0);
    cp_async_commit();
    for (int i = threadIdx.x; i < S; i += FWD_THREADS) sMask[i] = p.mask ? p.mask[(long long)b * S + i] * LOG2E : 0.f;

    const int r = lane >> 2, c = 2 * (lane & 3);
    const int q0 = qt * FWD_TQ + warp * 16 + r;                  // query rows q0 and q0 + 8 of this thread
    const unsigned long long seed = effective_seed(p.seed, p.seed_dev);
    const unsigned long long drop_row0 = ((unsigned long long)(b * p.A + h) * S + q0) * (unsigned long long)S;
    const unsigned long long drop_row1 = drop_row0 + 8ull * S;
    uint32_t qf[4][4];
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
        cp_async_wait<1>();
        __syncthreads();
        if (kt == 0) load_a_frags(sQ, warp * 16, lane, qf);
        float s[8][4];
        mma_abt(s, qf, sK + buf * TILE64_BYTES, lane);
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
#pragma unroll
            for (int g = 0; g < 2; ++g) {                                 // the two 32-key RNG groups of the tile
                const int key0 = kt * KT + g * 32;
                const uint4 ra = attn_dropout_block(seed, p.drop_stream, (drop_row0 + key0) >> 5);
                const uint4 rb = attn_dropout_block(seed, p.drop_stream, (drop_row1 + key0) >> 5);
#pragma unroll
                for (int w = 0; w < 4; ++w) {                             // column tile j = 4g + w holds pair word 4w + lane % 4
                    const uint32_t ka = attn_dropout_word(ra, 4 * w + (lane & 3), p.drop_k2);
                    const uint32_t kb = attn_dropout_word(rb, 4 * w + (lane & 3), p.drop_k2);
                    pr[4 * g + w][0] &= ka; pl[4 * g + w][0] &= ka;
                    pr[4 * g + w][1] &= kb; pl[4 * g + w][1] &= kb;
                }
            }
        }
        mma_pt(o, pr, sV + buf * TILE64_BYTES, lane);
        mma_pt(o, pl, sV + buf * TILE64_BYTES, lane);
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
// backward
// =================================================================================================
constexpr int BWD_WARPS = 4, BWD_THREADS = BWD_WARPS * 32;
// K, V (or Q, dO) of the CTA's own tile + a double-buffered pair of streamed tiles + per-row statistics / mask
constexpr int BWD_SMEM_BYTES = 2 * TILE64_BYTES + 4 * TILE64_BYTES + 4 * 512 * 4;

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

// dK, dV of one 64-key tile.  Thread layout of the transposed score tile: key rows kr, kr + 8 (kr = tile + warp*16 + lane/4),
// query columns 8j + 2(lane%4) + {0,1} of the current query tile.
//   P   = exp2(S * scale*log2e + mask*log2e - lse*log2e)          (bf16, as in forward)
//   P~  = keep-mask AND P
//   dS  = [ P~ * dP / (1-p) - P * delta ] * scale
//   dV += P~^T dO (times 1/(1-p) at the end),  dK += dS^T Q
__global__ void __launch_bounds__(BWD_THREADS)
attn_bwd_dkv_kernel(const AttnParams p) {
    extern __shared__ __align__(128) uint8_t smem[];
    const int S = p.S, nqt = S / KT;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int kt = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
    const uint32_t sK = smem_u32(smem), sV = sK + TILE64_BYTES, sQ = sV + TILE64_BYTES, sdO = sQ + 2 * TILE64_BYTES;
    float* sLse = reinterpret_cast<float*>(smem + 6 * TILE64_BYTES);          // [S] -lse*log2e
    float* sNd = sLse + 512;                                                   // [S] -delta*scale
    const long long ld = 3LL * p.H;
    const long long bh = (long long)b * p.A + h;

    load_tile<KT, BWD_THREADS>(sK, p.qkv, ld, p.H + h * HD, p, b, kt * KT);
    load_tile<KT, BWD_THREADS>(sV, p.qkv, ld, 2 * p.H + h * HD, p, b, kt * KT);
    load_tile<KT, BWD_THREADS>(sQ, p.qkv, ld, h * HD, p, b, 0);
    load_tile<KT, BWD_THREADS>(sdO, p.dctx, p.H, h * HD, p, b, 0);
    cp_async_commit();
    for (int i = threadIdx.x; i < S; i += BWD_THREADS) { sLse[i] = -p.lse[bh * S + i] * LOG2E; sNd[i] = -p.delta[bh * S + i] * p.scale; }

    const int r = lane >> 2, c = 2 * (lane & 3);
    const int kr = kt * KT + warp * 16 + r;                      // key rows kr and kr + 8 of this thread
    const float mk0 = p.mask ? p.mask[(long long)b * S + kr] * LOG2E : 0.f;
    const float mk1 = p.mask ? p.mask[(long long)b * S + kr + 8] * LOG2E : 0.f;
    const unsigned long long seed = effective_seed(p.seed, p.seed_dev);
    const float c1 = p.drop_scale * p.scale;
    uint32_t kf[4][4], vf[4][4];
    float dk[8][4], dv[8][4];
#pragma unroll
    for (int j = 0; j < 8; ++j) { dk[j][0] = dk[j][1] = dk[j][2] = dk[j][3] = 0.f; dv[j][0] = dv[j][1] = dv[j][2] = dv[j][3] = 0.f; }

    for (int qt = 0; qt < nqt; ++qt) {
        const int buf = qt & 1;
        if (qt + 1 < nqt) {
            load_tile<KT, BWD_THREADS>(sQ + (buf ^ 1) * TILE64_BYTES, p.qkv, ld, h * HD, p, b, (qt + 1) * KT);
            load_tile<KT, BWD_THREADS>(sdO + (buf ^ 1) * TILE64_BYTES, p.dctx, p.H, h * HD, p, b, (qt + 1) * KT);
        }
        cp_async_commit();
        cp_async_wait<1>();
        __syncthreads();
        if (qt == 0) { load_a_frags(sK, warp * 16, lane, kf); load_a_frags(sV, warp * 16, lane, vf); }
        const uint32_t tQ = sQ + buf * TILE64_BYTES, tdO = sdO + buf * TILE64_BYTES;
        float st[8][4], dpt[8][4];
        mma_abt(st, kf, tQ, lane);                               // S^T  = K Q^T
        mma_abt(dpt, vf, tdO, lane);                             // dP^T = V dO^T
        uint32_t pm[8][2], ds[8][2];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int q = qt * KT + j * 8 + c;                   // query columns q, q + 1
            const float2 nl = *reinterpret_cast<const float2*>(sLse + q);
            const float2 nd = *reinterpret_cast<const float2*>(sNd + q);
            const uint32_t p0 = pack_bf16(ex2(fmaf(st[j][0], p.scale_log2, mk0) + nl.x), ex2(fmaf(st[j][1], p.scale_log2, mk0) + nl.y));
            const uint32_t p1 = pack_bf16(ex2(fmaf(st[j][2], p.scale_log2, mk1) + nl.x), ex2(fmaf(st[j][3], p.scale_log2, mk1) + nl.y));
            uint32_t k0 = 0xFFFFFFFFu, k1 = 0xFFFFFFFFu;
            if (p.drop_on != 0u) {                               // keys kr and kr + 8 share the 32-element group of each query
                const unsigned long long row = (unsigned long long)(bh * S + q) * (unsigned long long)S;
                const uint4 ra = attn_dropout_block(seed, p.drop_stream, (row + kr) >> 5);
                const uint4 rb = attn_dropout_block(seed, p.drop_stream, (row + S + kr) >> 5);
                k0 = keep_half(ra, kr, p.drop_k2) | (keep_half(rb, kr, p.drop_k2) << 16);
                k1 = keep_half(ra, kr + 8, p.drop_k2) | (keep_half(rb, kr + 8, p.drop_k2) << 16);
            }
            pm[j][0] = p0 & k0; pm[j][1] = p1 & k1;
            const float2 f0 = unpack_bf16(p0), f1 = unpack_bf16(p1), g0 = unpack_bf16(pm[j][0]), g1 = unpack_bf16(pm[j][1]);
            ds[j][0] = pack_bf16(fmaf(g0.x * dpt[j][0], c1, f0.x * nd.x), fmaf(g0.y * dpt[j][1], c1, f0.y * nd.y));
            ds[j][1] = pack_bf16(fmaf(g1.x * dpt[j][2], c1, f1.x * nd.x), fmaf(g1.y * dpt[j][3], c1, f1.y * nd.y));
        }
        mma_pt(dv, pm, tdO, lane);                               // dV += P~^T dO
        mma_pt(dk, ds, tQ, lane);                                // dK += dS^T Q
        __syncthreads();
    }
    const int s_row0 = kt * KT + warp * 16;
    store_rows_bf16(p, dk, 1.0f, b, s_row0, p.H + h * HD, lane);
    store_rows_bf16(p, dv, p.drop_scale, b, s_row0, 2 * p.H + h * HD, lane);
}

// dQ of one 64-query tile: rows q, q + 8 (q = tile + warp*16 + lane/4), key columns of the current key tile.  dQ += dS K.
__global__ void __launch_bounds__(BWD_THREADS)
attn_bwd_dq_kernel(const AttnParams p) {
    extern __shared__ __align__(128) uint8_t smem[];
    const int S = p.S, nkt = S / KT;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int qt = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
    const uint32_t sQ = smem_u32(smem), sdO = sQ + TILE64_BYTES, sK = sdO + TILE64_BYTES, sV = sK + 2 * TILE64_BYTES;
    float* sMask = reinterpret_cast<float*>(smem + 6 * TILE64_BYTES);
    const long long ld = 3LL * p.H;
    const long long bh = (long long)b * p.A + h;

    load_tile<KT, BWD_THREADS>(sQ, p.qkv, ld, h * HD, p, b, qt * KT);
    load_tile<KT, BWD_THREADS>(sdO, p.dctx, p.H, h * HD, p, b, qt * KT);
    load_tile<KT, BWD_THREADS>(sK, p.qkv, ld, p.H + h * HD, p, b, 0);
    load_tile<KT, BWD_THREADS>(sV, p.qkv, ld, 2 * p.H + h * HD, p, b, 0);
    cp_async_commit();
    for (int i = threadIdx.x; i < S; i += BWD_THREADS) sMask[i] = p.mask ? p.mask[(long long)b * S + i] * LOG2E : 0.f;

    const int r = lane >> 2, c = 2 * (lane & 3);
    const int q0 = qt * KT + warp * 16 + r;
    const float nl0 = -p.lse[bh * S + q0] * LOG2E, nl1 = -p.lse[bh * S + q0 + 8] * LOG2E;
    const float nd0 = -p.delta[bh * S + q0] * p.scale, nd1 = -p.delta[bh * S + q0 + 8] * p.scale;
    const unsigned long long seed = effective_seed(p.seed, p.seed_dev);
    const unsigned long long drop_row0 = (unsigned long long)(bh * S + q0) * (unsigned long long)S;
    const unsigned long long drop_row1 = drop_row0 + 8ull * S;
    const float c1 = p.drop_scale * p.scale;
    uint32_t qf[4][4], of[4][4];
    float dq[8][4];
#pragma unroll
    for (int j = 0; j < 8; ++j) dq[j][0] = dq[j][1] = dq[j][2] = dq[j][3] = 0.f;

    for (int kt = 0; kt < nkt; ++kt) {
        const int buf = kt & 1;
        if (kt + 1 < nkt) {
            load_tile<KT, BWD_THREADS>(sK + (buf ^ 1) * TILE64_BYTES, p.qkv, ld, p.H + h * HD, p, b, (kt + 1) * KT);
            load_tile<KT, BWD_THREADS>(sV + (buf ^ 1) * TILE64_BYTES, p.qkv, ld, 2 * p.H + h * HD, p, b, (kt + 1) * KT);
        }
        cp_async_commit();
        cp_async_wait<1>();
        __syncthreads();
        if (kt == 0) { load_a_frags(sQ, warp * 16, lane, qf); load_a_frags(sdO, warp * 16, lane, of); }
        const uint32_t tK = sK + buf * TILE64_BYTES, tV = sV + buf * TILE64_BYTES;
        float s[8][4], dp[8][4];
        mma_abt(s, qf, tK, lane);                                // S  = Q K^T
        mma_abt(dp, of, tV, lane);                               // dP = dO V^T
        uint32_t km[8][2];
#pragma unroll
        for (int j = 0; j < 8; ++j) km[j][0] = km[j][1] = 0xFFFFFFFFu;
        if (p.drop_on != 0u) {
#pragma unroll
            for (int g = 0; g < 2; ++g) {
                const int key0 = kt * KT + g * 32;
                const uint4 ra = attn_dropout_block(seed, p.drop_stream, (drop_row0 + key0) >> 5);
                const uint4 rb = attn_dropout_block(seed, p.drop_stream, (drop_row1 + key0) >> 5);
#pragma unroll
                for (int w = 0; w < 4; ++w) {
                    km[4 * g + w][0] = attn_dropout_word(ra, 4 * w + (lane & 3), p.drop_k2);
                    km[4 * g + w][1] = attn_dropout_word(rb, 4 * w + (lane & 3), p.drop_k2);
                }
            }
        }
        uint32_t ds[8][2];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const float2 mk = *reinterpret_cast<const float2*>(sMask + kt * KT + j * 8 + c);
            const uint32_t p0 = pack_bf16(ex2(fmaf(s[j][0], p.scale_log2, mk.x) + nl0), ex2(fmaf(s[j][1], p.scale_log2, mk.y) + nl0));
            const uint32_t p1 = pack_bf16(ex2(fmaf(s[j][2], p.scale_log2, mk.x) + nl1), ex2(fmaf(s[j][3], p.scale_log2, mk.y) + nl1));
            const float2 f0 = unpack_bf16(p0), f1 = unpack_bf16(p1), g0 = unpack_bf16(p0 & km[j][0]), g1 = unpack_bf16(p1 & km[j][1]);
            ds[j][0] = pack_bf16(fmaf(g0.x * dp[j][0], c1, f0.x * nd0), fmaf(g0.y * dp[j][1], c1, f0.y * nd0));
            ds[j][1] = pack_bf16(fmaf(g1.x * dp[j][2], c1, f1.x * nd1), fmaf(g1.y * dp[j][3], c1, f1.y * nd1));
        }
        mma_pt(dq, ds, tK, lane);                                // dQ += dS K
        __syncthreads();
    }
    store_rows_bf16(p, dq, 1.0f, b, qt * KT + warp * 16, h * HD, lane);
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
    int rc = ensure_smem_attr(attn_bwd_dkv_kernel, attr_kv, BWD_SMEM_BYTES);
    if (rc != DLE_OK) return rc;
    rc = ensure_smem_attr(attn_bwd_dq_kernel, attr_q, BWD_SMEM_BYTES);
    if (rc != DLE_OK) return rc;
    attn_bwd_dkv_kernel<<<dim3(S / KT, A, B), BWD_THREADS, BWD_SMEM_BYTES, st>>>(p);
    DLE_LAUNCH_CHECK();
    attn_bwd_dq_kernel<<<dim3(S / KT, A, B), BWD_THREADS, BWD_SMEM_BYTES, st>>>(p);
    DLE_LAUNCH_CHECK();
    return DLE_OK;
}
