// Distillation losses for sm_90a without the [B, A, S, S] tensors the reference materialises.
//
// Relation-KL: for each (b, h) the student logits s = scale_s * X_s Y_s^T (+ mask) and the teacher logits t = scale_t * X_t Y_t^T
// (+ mask) are [S, S]; the loss is sum over all B*A*S query rows of KL(softmax(t) || softmax(s)), times a normalisation factor.
//   attention scores : X = Q, Y = K (column blocks h and A + h of the packed qkv [T, 3H]), additive mask, and the reference's
//                      where(x <= -100, 0, x) on both logit sets (losses.py:80-85)
//   value relation   : X = Y = ctx (column block h of [T, H]), no mask (losses.py:41-61)
// Operands are bf16 head slices (head dim 64) of token-row matrices, padded [B, S] grid in either token order, S % 64 == 0, S <= 512.
//
// Forward : one CTA (one warpgroup) per (b, h, 64-query tile).  X_s and X_t tiles stay resident, Y_s / Y_t tiles of 64 keys stream
//           through double-buffered cp.async into 128B-swizzled shared memory; both products on wgmma m64n64k16 (fp32 accumulators).
//           Per row, online max and sum of both distributions and the running cross term sum e^(t - m_t) (t - s), rescaled like the
//           attention kernels' O.  Row KL = cross / Z_t - lse_t + lse_s.  lse_s / lse_t [B, A, S] are kept for backward; each CTA
//           writes one fp32 partial (its rows summed in a fixed order) and a one-block finalize launch sums the partials in a fixed
//           order: no atomics, bitwise reproducible, capturable.
// Backward: dS = g * norm * scale_s * (p_s - p_t), exactly 0 where the where-rule replaced the logit.  No delta pass is needed.
//             dX : one CTA per (b, h, 64-query tile) walks the key tiles, dX += dS Y_s
//             dY : one CTA per (b, h, 64-key tile) walks the query tiles, dY += dS^T X_s
//           Each output element has exactly one owner.  With X = Y (value relation) the dY launch adds onto the dX launch's output.
// Cosine rows: mean over rows of 1 - cos(pred, target) with torch's CosineEmbeddingLoss eps (losses.py:63-70), forward and backward.
#include "common.cuh"
#include "../../include/dle_b200.h"

namespace dle {
namespace distill {

constexpr int HD = 64;
constexpr int KT = 64;
constexpr int TILE_BYTES = KT * HD * 2;
constexpr int THREADS = 128;
constexpr float LOG2E = 1.4426950408889634f;
constexpr float WHERE_BOUND = -100.f;
constexpr int SMEM_BYTES = 1024 /*alignment*/ + 6 * TILE_BYTES /*X_s, X_t, Y_s x 2, Y_t x 2*/ + 4 * 512 * 4 /*masks or lse*/;

__device__ __forceinline__ float ex2(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
__device__ __forceinline__ uint32_t sw(int r, int ch) { return (uint32_t)(r * 128 + ((ch ^ (r & 7)) << 4)); }
__device__ __forceinline__ uint8_t* smem_1k(uint8_t* smem) {
    return smem + (((smem_u32(smem) + 1023u) & ~1023u) - smem_u32(smem));
}

struct RelKLParams {
    const bf16* xs; const bf16* ys; const bf16* xt; const bf16* yt;   // column block of head 0 of each operand
    long long ld_s, ld_t;                                             // row strides (elements) of the student / teacher matrices
    const float* mask_s; const float* mask_t;                         // [B, S] additive or null
    float scale_s, scale_t;
    int where_rule;
    int B, S, A, tok_stride_s, tok_stride_b;
    float* lse_s; float* lse_t;                                       // [B, A, S]
    float* partial;                                                   // [B * A * S / 64]
    const float* gscale; float norm;                                  // backward: dL/dloss (device scalar) and the 1/(B*A*S) factor
    bf16* dx; bf16* dy; long long ld_d;                               // backward outputs: column block of head 0
    bf16* dzero;                                                      // backward: column block of head 0 to zero-fill (or null)
    int accumulate_dy;                                                // dY adds onto dx's values (value relation: X = Y)
};

__device__ __forceinline__ long long tok_row(const RelKLParams& p, int b, int s) {
    return (long long)b * p.tok_stride_b + (long long)s * p.tok_stride_s;
}
// rows [s0, s0 + 64) of head h's 64 columns of a token-row matrix -> swizzled smem tile
__device__ __forceinline__ void load_tile(uint32_t dst, const bf16* base, long long ld, const RelKLParams& p, int b, int h, int s0) {
#pragma unroll
    for (int i = 0; i < KT * 8 / THREADS; ++i) {
        const int idx = threadIdx.x + i * THREADS, r = idx >> 3, ch = idx & 7;
        cp_async16(dst + sw(r, ch), base + tok_row(p, b, s0 + r) * ld + h * HD + ch * 8);
    }
}
template <int N> __device__ __forceinline__ void tiles_ready() {
    cp_async_wait<N>();
    fence_proxy_async_smem();
    __syncthreads();
}
__device__ __forceinline__ void wg_abt(float (&acc)[8][4], uint32_t a, uint32_t t) {
#pragma unroll
    for (int kk = 0; kk < 4; ++kk)
        wgmma_m64n64k16<0, 0>(acc, make_wgmma_desc_sw128(a + kk * 32, 16, 1024), make_wgmma_desc_sw128(t + kk * 32, 16, 1024), kk > 0 ? 1u : 0u);
}
__device__ __forceinline__ void wg_pt(float (&acc)[8][4], const uint32_t (&pr)[8][2], uint32_t t) {
#pragma unroll
    for (int kk = 0; kk < 4; ++kk)
        wgmma_m64n64k16_rs<1>(acc, pr[2 * kk][0], pr[2 * kk][1], pr[2 * kk + 1][0], pr[2 * kk + 1][1],
                              make_wgmma_desc_sw128(t + kk * 16 * 128, TILE_BYTES, 1024));
}
// one logit: fma(acc, scale, mask), then the where rule; `sub` reports a substituted logit
__device__ __forceinline__ float logit(float acc, float scale, float mk, int where_rule, bool& sub) {
    const float v = fmaf(acc, scale, mk);
    sub = where_rule && v <= WHERE_BOUND;
    return sub ? 0.f : v;
}

// =================================================================================================
// forward
// =================================================================================================
__global__ void __launch_bounds__(THREADS)
relkl_fwd_kernel(const RelKLParams p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_1k(smem_raw);
    const int S = p.S, nkt = S / KT;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int qt = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
    const uint32_t sXs = smem_u32(smem), sXt = sXs + TILE_BYTES, sYs = sXt + TILE_BYTES, sYt = sYs + 2 * TILE_BYTES;
    float* sMs = reinterpret_cast<float*>(smem + 6 * TILE_BYTES);
    float* sMt = sMs + 512;
    float* sRed = sMt + 512;                                          // [4] per-warp sums

    load_tile(sXs, p.xs, p.ld_s, p, b, h, qt * KT);
    load_tile(sXt, p.xt, p.ld_t, p, b, h, qt * KT);
    load_tile(sYs, p.ys, p.ld_s, p, b, h, 0);
    load_tile(sYt, p.yt, p.ld_t, p, b, h, 0);
    cp_async_commit();
    for (int i = threadIdx.x; i < S; i += THREADS) {
        sMs[i] = p.mask_s ? p.mask_s[(long long)b * S + i] : 0.f;
        sMt[i] = p.mask_t ? p.mask_t[(long long)b * S + i] : 0.f;
    }

    const int r = lane >> 2, c = 2 * (lane & 3);
    const int q0 = qt * KT + warp * 16 + r;                            // query rows q0 and q0 + 8 of this thread
    // per row i in {0, 1}: running maxima, sums of e^(x - m) (this thread's columns) and the cross term
    float ms[2] = {-INFINITY, -INFINITY}, mt[2] = {-INFINITY, -INFINITY};
    float ls[2] = {0.f, 0.f}, lt[2] = {0.f, 0.f}, cr[2] = {0.f, 0.f};

    for (int kt = 0; kt < nkt; ++kt) {
        const int buf = kt & 1;
        if (kt + 1 < nkt) {
            load_tile(sYs + (buf ^ 1) * TILE_BYTES, p.ys, p.ld_s, p, b, h, (kt + 1) * KT);
            load_tile(sYt + (buf ^ 1) * TILE_BYTES, p.yt, p.ld_t, p, b, h, (kt + 1) * KT);
        }
        cp_async_commit();
        tiles_ready<1>();
        float s[8][4], t[8][4];
        wgmma_fence();
        wg_abt(s, sXs, sYs + buf * TILE_BYTES);
        wg_abt(t, sXt, sYt + buf * TILE_BYTES);
        wgmma_commit();
        wgmma_wait<0>();
        fence_regs(s); fence_regs(t);
        float mxs[2] = {-INFINITY, -INFINITY}, mxt[2] = {-INFINITY, -INFINITY};
#pragma unroll
        for (int j = 0; j < 8; ++j) {
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int key = kt * KT + j * 8 + c + (e & 1);
                bool sub;
                s[j][e] = logit(s[j][e], p.scale_s, sMs[key], p.where_rule, sub);
                t[j][e] = logit(t[j][e], p.scale_t, sMt[key], p.where_rule, sub);
                mxs[e >> 1] = fmaxf(mxs[e >> 1], s[j][e]);
                mxt[e >> 1] = fmaxf(mxt[e >> 1], t[j][e]);
            }
        }
#pragma unroll
        for (int i = 0; i < 2; ++i) {
#pragma unroll
            for (int off = 1; off < 4; off <<= 1) {
                mxs[i] = fmaxf(mxs[i], __shfl_xor_sync(0xffffffffu, mxs[i], off));
                mxt[i] = fmaxf(mxt[i], __shfl_xor_sync(0xffffffffu, mxt[i], off));
            }
            const float ns = fmaxf(ms[i], mxs[i]), nt = fmaxf(mt[i], mxt[i]);
            const float as = ex2((ms[i] - ns) * LOG2E), at = ex2((mt[i] - nt) * LOG2E);     // 0 on the first tile
            ls[i] *= as; lt[i] *= at; cr[i] *= at;
            ms[i] = ns; mt[i] = nt;
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) {
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int i = e >> 1;
                const float es = ex2((s[j][e] - ms[i]) * LOG2E), et = ex2((t[j][e] - mt[i]) * LOG2E);
                ls[i] += es; lt[i] += et;
                cr[i] = fmaf(et, t[j][e] - s[j][e], cr[i]);
            }
        }
        __syncthreads();                                              // buffer `buf` is refilled at the next iteration
    }
    float kl = 0.f;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
#pragma unroll
        for (int off = 1; off < 4; off <<= 1) {
            ls[i] += __shfl_xor_sync(0xffffffffu, ls[i], off);
            lt[i] += __shfl_xor_sync(0xffffffffu, lt[i], off);
            cr[i] += __shfl_xor_sync(0xffffffffu, cr[i], off);
        }
        const float lse_s = ms[i] + logf(ls[i]), lse_t = mt[i] + logf(lt[i]);
        kl += cr[i] / lt[i] - lse_t + lse_s;
        if ((lane & 3) == 0) {
            const long long o = ((long long)b * p.A + h) * S + q0 + 8 * i;
            p.lse_s[o] = lse_s;
            p.lse_t[o] = lse_t;
        }
    }
    // rows of the warp: lanes 0, 4, ..., 28 hold them; a fixed shuffle tree, then the four warps in order
    kl = (lane & 3) == 0 ? kl : 0.f;
    kl = warp_sum(kl);
    if (lane == 0) sRed[warp] = kl;
    __syncthreads();
    if (threadIdx.x == 0)
        p.partial[((long long)b * p.A + h) * (S / KT) + qt] = (sRed[0] + sRed[1]) + (sRed[2] + sRed[3]);
}

// out[0] = norm * sum of part[0 .. n), in a fixed order (one block)
constexpr int FIN_THREADS = 256;
__global__ void __launch_bounds__(FIN_THREADS)
sum_partials_kernel(const float* __restrict__ part, long long n, float norm, float* __restrict__ out) {
    __shared__ float red[FIN_THREADS / 32];
    float acc = 0.f;
    for (long long i = threadIdx.x; i < n; i += FIN_THREADS) acc += part[i];
    acc = warp_sum(acc);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        float s = 0.f;
#pragma unroll
        for (int w = 0; w < FIN_THREADS / 32; ++w) s += red[w];
        out[0] = s * norm;
    }
}

// bf16 rows [r0, r0 + 16) x 64 columns of a fragment accumulator -> out (head column block h); optionally added onto out's values
__device__ __forceinline__ void store_rows(const RelKLParams& p, bf16* base, const float (&acc)[8][4], int b, int h, int s_row0,
                                           bool accumulate, int lane) {
    const int r = lane >> 2, c = 2 * (lane & 3);
    bf16* o0 = base + tok_row(p, b, s_row0 + r) * p.ld_d + h * HD;
    bf16* o1 = base + tok_row(p, b, s_row0 + r + 8) * p.ld_d + h * HD;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        float a0 = acc[j][0], a1 = acc[j][1], a2 = acc[j][2], a3 = acc[j][3];
        if (accumulate) {
            const float2 f0 = unpack_bf16(*reinterpret_cast<const uint32_t*>(o0 + j * 8 + c));
            const float2 f1 = unpack_bf16(*reinterpret_cast<const uint32_t*>(o1 + j * 8 + c));
            a0 += f0.x; a1 += f0.y; a2 += f1.x; a3 += f1.y;
        }
        *reinterpret_cast<uint32_t*>(o0 + j * 8 + c) = pack_bf16(a0, a1);
        *reinterpret_cast<uint32_t*>(o1 + j * 8 + c) = pack_bf16(a2, a3);
    }
}

// =================================================================================================
// backward, dX: rows q, q + 8 (q = tile + warp*16 + lane/4) against the key columns of each key tile
// =================================================================================================
__global__ void __launch_bounds__(THREADS)
relkl_bwd_dx_kernel(const RelKLParams p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_1k(smem_raw);
    const int S = p.S, nkt = S / KT;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int qt = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
    const uint32_t sXs = smem_u32(smem), sXt = sXs + TILE_BYTES, sYs = sXt + TILE_BYTES, sYt = sYs + 2 * TILE_BYTES;
    float* sMs = reinterpret_cast<float*>(smem + 6 * TILE_BYTES);
    float* sMt = sMs + 512;

    load_tile(sXs, p.xs, p.ld_s, p, b, h, qt * KT);
    load_tile(sXt, p.xt, p.ld_t, p, b, h, qt * KT);
    load_tile(sYs, p.ys, p.ld_s, p, b, h, 0);
    load_tile(sYt, p.yt, p.ld_t, p, b, h, 0);
    cp_async_commit();
    for (int i = threadIdx.x; i < S; i += THREADS) {
        sMs[i] = p.mask_s ? p.mask_s[(long long)b * S + i] : 0.f;
        sMt[i] = p.mask_t ? p.mask_t[(long long)b * S + i] : 0.f;
    }
    const int r = lane >> 2, c = 2 * (lane & 3);
    const int q0 = qt * KT + warp * 16 + r;
    const long long bh = (long long)b * p.A + h;
    const float nls[2] = {-p.lse_s[bh * S + q0] * LOG2E, -p.lse_s[bh * S + q0 + 8] * LOG2E};
    const float nlt[2] = {-p.lse_t[bh * S + q0] * LOG2E, -p.lse_t[bh * S + q0 + 8] * LOG2E};
    const float coef = *p.gscale * p.norm * p.scale_s;
    float dx[8][4];
#pragma unroll
    for (int j = 0; j < 8; ++j) dx[j][0] = dx[j][1] = dx[j][2] = dx[j][3] = 0.f;

    for (int kt = 0; kt < nkt; ++kt) {
        const int buf = kt & 1;
        if (kt + 1 < nkt) {
            load_tile(sYs + (buf ^ 1) * TILE_BYTES, p.ys, p.ld_s, p, b, h, (kt + 1) * KT);
            load_tile(sYt + (buf ^ 1) * TILE_BYTES, p.yt, p.ld_t, p, b, h, (kt + 1) * KT);
        }
        cp_async_commit();
        tiles_ready<1>();
        const uint32_t tYs = sYs + buf * TILE_BYTES;
        float s[8][4], t[8][4];
        wgmma_fence();
        wg_abt(s, sXs, tYs);
        wg_abt(t, sXt, sYt + buf * TILE_BYTES);
        wgmma_commit();
        wgmma_wait<0>();
        fence_regs(s); fence_regs(t);
        uint32_t ds[8][2];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            float d[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int key = kt * KT + j * 8 + c + (e & 1), i = e >> 1;
                bool sub_s, sub_t;
                const float vs = logit(s[j][e], p.scale_s, sMs[key], p.where_rule, sub_s);
                const float vt = logit(t[j][e], p.scale_t, sMt[key], p.where_rule, sub_t);
                const float ps = ex2(fmaf(vs, LOG2E, nls[i])), pt = ex2(fmaf(vt, LOG2E, nlt[i]));
                d[e] = sub_s ? 0.f : (ps - pt) * coef;
            }
            ds[j][0] = pack_bf16(d[0], d[1]);
            ds[j][1] = pack_bf16(d[2], d[3]);
        }
        fence_regs(dx);
        wgmma_fence();
        wg_pt(dx, ds, tYs);                                           // dX += dS Y_s
        wgmma_commit();
        wgmma_wait<0>();
        fence_regs(dx); fence_regs(ds);
        __syncthreads();
    }
    store_rows(p, p.dx, dx, b, h, qt * KT + warp * 16, false, lane);
}

// =================================================================================================
// backward, dY: key rows k, k + 8 (k = tile + warp*16 + lane/4) against the query columns of each query tile (transposed scores)
// =================================================================================================
__global__ void __launch_bounds__(THREADS)
relkl_bwd_dy_kernel(const RelKLParams p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_1k(smem_raw);
    const int S = p.S, nqt = S / KT;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int kt = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
    const uint32_t sYs = smem_u32(smem), sYt = sYs + TILE_BYTES, sXs = sYt + TILE_BYTES, sXt = sXs + 2 * TILE_BYTES;
    float* sLs = reinterpret_cast<float*>(smem + 6 * TILE_BYTES);     // [S] -lse_s * log2e
    float* sLt = sLs + 512;                                           // [S] -lse_t * log2e
    const long long bh = (long long)b * p.A + h;

    load_tile(sYs, p.ys, p.ld_s, p, b, h, kt * KT);
    load_tile(sYt, p.yt, p.ld_t, p, b, h, kt * KT);
    load_tile(sXs, p.xs, p.ld_s, p, b, h, 0);
    load_tile(sXt, p.xt, p.ld_t, p, b, h, 0);
    cp_async_commit();
    for (int i = threadIdx.x; i < S; i += THREADS) { sLs[i] = -p.lse_s[bh * S + i] * LOG2E; sLt[i] = -p.lse_t[bh * S + i] * LOG2E; }

    const int r = lane >> 2, c = 2 * (lane & 3);
    const int k0 = kt * KT + warp * 16 + r;                           // key rows k0 and k0 + 8 of this thread
    const float mks[2] = {p.mask_s ? p.mask_s[(long long)b * S + k0] : 0.f, p.mask_s ? p.mask_s[(long long)b * S + k0 + 8] : 0.f};
    const float mkt[2] = {p.mask_t ? p.mask_t[(long long)b * S + k0] : 0.f, p.mask_t ? p.mask_t[(long long)b * S + k0 + 8] : 0.f};
    const float coef = *p.gscale * p.norm * p.scale_s;
    float dy[8][4];
#pragma unroll
    for (int j = 0; j < 8; ++j) dy[j][0] = dy[j][1] = dy[j][2] = dy[j][3] = 0.f;

    for (int qt = 0; qt < nqt; ++qt) {
        const int buf = qt & 1;
        if (qt + 1 < nqt) {
            load_tile(sXs + (buf ^ 1) * TILE_BYTES, p.xs, p.ld_s, p, b, h, (qt + 1) * KT);
            load_tile(sXt + (buf ^ 1) * TILE_BYTES, p.xt, p.ld_t, p, b, h, (qt + 1) * KT);
        }
        cp_async_commit();
        tiles_ready<1>();
        const uint32_t tXs = sXs + buf * TILE_BYTES;
        float s[8][4], t[8][4];
        wgmma_fence();
        wg_abt(s, sYs, tXs);                                          // S^T = Y_s X_s^T
        wg_abt(t, sYt, sXt + buf * TILE_BYTES);
        wgmma_commit();
        wgmma_wait<0>();
        fence_regs(s); fence_regs(t);
        uint32_t ds[8][2];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            float d[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int q = qt * KT + j * 8 + c + (e & 1), i = e >> 1;
                bool sub_s, sub_t;
                const float vs = logit(s[j][e], p.scale_s, mks[i], p.where_rule, sub_s);
                const float vt = logit(t[j][e], p.scale_t, mkt[i], p.where_rule, sub_t);
                const float ps = ex2(fmaf(vs, LOG2E, sLs[q])), pt = ex2(fmaf(vt, LOG2E, sLt[q]));
                d[e] = sub_s ? 0.f : (ps - pt) * coef;
            }
            ds[j][0] = pack_bf16(d[0], d[1]);
            ds[j][1] = pack_bf16(d[2], d[3]);
        }
        fence_regs(dy);
        wgmma_fence();
        wg_pt(dy, ds, tXs);                                           // dY += dS^T X_s
        wgmma_commit();
        wgmma_wait<0>();
        fence_regs(dy); fence_regs(ds);
        __syncthreads();
    }
    const int s_row0 = kt * KT + warp * 16;
    store_rows(p, p.dy, dy, b, h, s_row0, p.accumulate_dy != 0, lane);
    if (p.dzero != nullptr) {                                         // the V block of a packed qkv gradient: exactly 0
        const float zero[8][4] = {};
        store_rows(p, p.dzero, zero, b, h, s_row0, false, lane);
    }
}

// =================================================================================================
// cosine rows: loss = mean_r (1 - cos(x_r, y_r)), cos = <x, y> / sqrt((|x|^2 + eps)(|y|^2 + eps)); one warp per row
// =================================================================================================
constexpr float COS_EPS = 1e-12f;           // EPSILON of torch's cosine_embedding_loss
constexpr int COS_THREADS = 256, COS_ROWS_PER_BLOCK = 64;

__device__ __forceinline__ void row_dots(const bf16* x, const bf16* y, int H, int lane, float& xy, float& xx, float& yy) {
    xy = xx = yy = 0.f;
    for (int c = lane * 8; c < H; c += 256) {
        const uint4 ux = ld_global_nc_v4(x + c), uy = ld_global_nc_v4(y + c);
        const uint32_t ax[4] = {ux.x, ux.y, ux.z, ux.w}, ay[4] = {uy.x, uy.y, uy.z, uy.w};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const float2 fx = unpack_bf16(ax[k]), fy = unpack_bf16(ay[k]);
            xy = fmaf(fx.x, fy.x, fmaf(fx.y, fy.y, xy));
            xx = fmaf(fx.x, fx.x, fmaf(fx.y, fx.y, xx));
            yy = fmaf(fy.x, fy.x, fmaf(fy.y, fy.y, yy));
        }
    }
    xy = warp_sum(xy); xx = warp_sum(xx); yy = warp_sum(yy);
}

// one partial per block: the sum of 1 - cos over its COS_ROWS_PER_BLOCK rows, warps in order
__global__ void __launch_bounds__(COS_THREADS)
cosine_rows_fwd_kernel(const bf16* __restrict__ x, long long ldx, const bf16* __restrict__ y, long long ldy, long long rows, int H,
                       float* __restrict__ partial) {
    __shared__ float red[COS_THREADS / 32];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    float acc = 0.f;
    for (int i = warp; i < COS_ROWS_PER_BLOCK; i += COS_THREADS / 32) {
        const long long row = (long long)blockIdx.x * COS_ROWS_PER_BLOCK + i;
        if (row >= rows) break;
        float xy, xx, yy;
        row_dots(x + row * ldx, y + row * ldy, H, lane, xy, xx, yy);
        acc += 1.f - xy / sqrtf((xx + COS_EPS) * (yy + COS_EPS));
    }
    if (lane == 0) red[warp] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        float s = 0.f;
#pragma unroll
        for (int w = 0; w < COS_THREADS / 32; ++w) s += red[w];
        partial[blockIdx.x] = s;
    }
}

// dx_r = -(g / rows) * (y_r / sqrt((|x|^2 + eps)(|y|^2 + eps)) - cos * x_r / (|x|^2 + eps))
__global__ void __launch_bounds__(COS_THREADS)
cosine_rows_bwd_kernel(const bf16* __restrict__ x, long long ldx, const bf16* __restrict__ y, long long ldy, long long rows, int H,
                       const float* __restrict__ gscale, float norm, bf16* __restrict__ dx, long long ldd) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const float g = -*gscale * norm;
    for (long long row = (long long)blockIdx.x * (COS_THREADS / 32) + warp; row < rows; row += (long long)gridDim.x * (COS_THREADS / 32)) {
        const bf16* xr = x + row * ldx; const bf16* yr = y + row * ldy;
        float xy, xx, yy;
        row_dots(xr, yr, H, lane, xy, xx, yy);
        const float inv = rsqrtf((xx + COS_EPS) * (yy + COS_EPS));
        const float cy = g * inv, cx = -g * xy * inv / (xx + COS_EPS);
        for (int c = lane * 8; c < H; c += 256) {
            const uint4 ux = ld_global_nc_v4(xr + c), uy = ld_global_nc_v4(yr + c);
            const uint32_t ax[4] = {ux.x, ux.y, ux.z, ux.w}, ay[4] = {uy.x, uy.y, uy.z, uy.w};
            uint32_t o[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const float2 fx = unpack_bf16(ax[k]), fy = unpack_bf16(ay[k]);
                o[k] = pack_bf16(fmaf(cy, fy.x, cx * fx.x), fmaf(cy, fy.y, cx * fx.y));
            }
            st_global_v4(dx + row * ldd + c, o[0], o[1], o[2], o[3]);
        }
    }
}

// =================================================================================================
// dst[r, c] = bf16(dst + src) over [rows, cols]; column sums of src added to colsum (fp32, atomics) when given
// =================================================================================================
constexpr int ADD_ROWS_PER_THREAD = 32;
__global__ void __launch_bounds__(256)
add_rows_bf16_kernel(bf16* __restrict__ dst, long long ldd, const bf16* __restrict__ src, long long lds, long long rows, int cols,
                     float* __restrict__ colsum) {
    const int c = (blockIdx.x * 32 + threadIdx.x) * 2;               // column pair
    const long long r0 = ((long long)blockIdx.y * 8 + threadIdx.y) * ADD_ROWS_PER_THREAD;
    if (c >= cols) return;
    float s0 = 0.f, s1 = 0.f;
    for (int i = 0; i < ADD_ROWS_PER_THREAD; ++i) {
        const long long r = r0 + i;
        if (r >= rows) break;
        const float2 a = unpack_bf16(*reinterpret_cast<const uint32_t*>(src + r * lds + c));
        uint32_t* d = reinterpret_cast<uint32_t*>(dst + r * ldd + c);
        const float2 v = unpack_bf16(*d);
        *d = pack_bf16(v.x + a.x, v.y + a.y);
        s0 += a.x; s1 += a.y;
    }
    if (colsum != nullptr) { atomicAdd(colsum + c, s0); atomicAdd(colsum + c + 1, s1); }
}

}  // namespace distill
}  // namespace dle

using namespace dle;
using namespace dle::distill;

static bool aligned16(const void* x) { return (reinterpret_cast<uintptr_t>(x) & 15) == 0; }
static int smem_attr_once(const void* kern) {
    static int done[64][3] = {};
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return DLE_ERR_CUDA;
    const void* kerns[3] = {reinterpret_cast<const void*>(relkl_fwd_kernel), reinterpret_cast<const void*>(relkl_bwd_dx_kernel),
                            reinterpret_cast<const void*>(relkl_bwd_dy_kernel)};
    for (int i = 0; i < 3; ++i) {
        if (kerns[i] != kern || done[dev][i]) continue;
        if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES) != cudaSuccess) return DLE_ERR_CUDA;
        done[dev][i] = 1;
    }
    return DLE_OK;
}
static bool relkl_args_ok(const void* xs, const void* ys, const void* xt, const void* yt, int64_t ld_s, int64_t ld_t, int B, int S, int A) {
    return xs && ys && xt && yt && B > 0 && B <= 65535 && A > 0 && A <= 65535 && S > 0 && S % 64 == 0 && S <= 512 &&
           ld_s >= (int64_t)A * 64 && ld_t >= (int64_t)A * 64 && ld_s % 8 == 0 && ld_t % 8 == 0 &&
           aligned16(xs) && aligned16(ys) && aligned16(xt) && aligned16(yt);
}
static void relkl_common(RelKLParams& p, const void* xs, const void* ys, const void* xt, const void* yt, int64_t ld_s, int64_t ld_t,
                         const float* mask_s, const float* mask_t, float scale_s, float scale_t, int32_t where_rule, int B, int S, int A,
                         int seq_first, float* lse_s, float* lse_t) {
    p = RelKLParams{};
    p.xs = reinterpret_cast<const bf16*>(xs); p.ys = reinterpret_cast<const bf16*>(ys);
    p.xt = reinterpret_cast<const bf16*>(xt); p.yt = reinterpret_cast<const bf16*>(yt);
    p.ld_s = ld_s; p.ld_t = ld_t; p.mask_s = mask_s; p.mask_t = mask_t;
    p.scale_s = scale_s; p.scale_t = scale_t; p.where_rule = where_rule ? 1 : 0;
    p.B = B; p.S = S; p.A = A;
    p.tok_stride_s = seq_first ? B : 1; p.tok_stride_b = seq_first ? 1 : S;
    p.lse_s = lse_s; p.lse_t = lse_t;
}

extern "C" int dle_relkl_partials(int32_t B, int32_t S, int32_t A) {
    if (B <= 0 || A <= 0 || S <= 0 || S % 64 != 0) return DLE_ERR_INVALID;
    return B * A * (S / 64);
}

extern "C" int dle_relkl_fwd(const void* xs, const void* ys, const void* xt, const void* yt, int64_t ld_s, int64_t ld_t,
                             const float* mask_s, const float* mask_t, float scale_s, float scale_t, int32_t where_rule, int32_t B,
                             int32_t S, int32_t A, int32_t seq_first, float norm, float* lse_s, float* lse_t, float* partial, float* loss,
                             void* stream) {
    DLE_CHECK_ARG(relkl_args_ok(xs, ys, xt, yt, ld_s, ld_t, B, S, A) && lse_s && lse_t && partial && loss);
    RelKLParams p;
    relkl_common(p, xs, ys, xt, yt, ld_s, ld_t, mask_s, mask_t, scale_s, scale_t, where_rule, B, S, A, seq_first, lse_s, lse_t);
    p.partial = partial;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    int rc = smem_attr_once(reinterpret_cast<const void*>(relkl_fwd_kernel));
    if (rc != DLE_OK) return rc;
    relkl_fwd_kernel<<<dim3(S / KT, A, B), THREADS, SMEM_BYTES, st>>>(p);
    DLE_LAUNCH_CHECK();
    sum_partials_kernel<<<1, FIN_THREADS, 0, st>>>(partial, (long long)B * A * (S / KT), norm, loss);
    DLE_LAUNCH_CHECK();
    return DLE_OK;
}

extern "C" int dle_relkl_bwd(const void* xs, const void* ys, const void* xt, const void* yt, int64_t ld_s, int64_t ld_t,
                             const float* mask_s, const float* mask_t, float scale_s, float scale_t, int32_t where_rule, int32_t B,
                             int32_t S, int32_t A, int32_t seq_first, const float* lse_s, const float* lse_t, const float* grad_scale,
                             float norm, void* dx, void* dy, void* dzero, int64_t ld_d, void* stream) {
    DLE_CHECK_ARG(relkl_args_ok(xs, ys, xt, yt, ld_s, ld_t, B, S, A) && lse_s && lse_t && grad_scale && dx && dy);
    DLE_CHECK_ARG(ld_d >= (int64_t)A * 64 && ld_d % 8 == 0 && aligned16(dx) && aligned16(dy) && (dzero == nullptr || aligned16(dzero)));
    RelKLParams p;
    relkl_common(p, xs, ys, xt, yt, ld_s, ld_t, mask_s, mask_t, scale_s, scale_t, where_rule, B, S, A, seq_first,
                 const_cast<float*>(lse_s), const_cast<float*>(lse_t));
    p.gscale = grad_scale; p.norm = norm;
    p.dx = reinterpret_cast<bf16*>(dx); p.dy = reinterpret_cast<bf16*>(dy); p.dzero = reinterpret_cast<bf16*>(dzero); p.ld_d = ld_d;
    p.accumulate_dy = dx == dy ? 1 : 0;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    int rc = smem_attr_once(reinterpret_cast<const void*>(relkl_bwd_dx_kernel));
    if (rc != DLE_OK) return rc;
    rc = smem_attr_once(reinterpret_cast<const void*>(relkl_bwd_dy_kernel));
    if (rc != DLE_OK) return rc;
    relkl_bwd_dx_kernel<<<dim3(S / KT, A, B), THREADS, SMEM_BYTES, st>>>(p);
    DLE_LAUNCH_CHECK();
    relkl_bwd_dy_kernel<<<dim3(S / KT, A, B), THREADS, SMEM_BYTES, st>>>(p);
    DLE_LAUNCH_CHECK();
    return DLE_OK;
}

extern "C" int dle_cosine_rows_partials(int64_t rows) {
    if (rows <= 0) return DLE_ERR_INVALID;
    return (int)((rows + COS_ROWS_PER_BLOCK - 1) / COS_ROWS_PER_BLOCK);
}

extern "C" int dle_cosine_rows_fwd(const void* x, int64_t ldx, const void* y, int64_t ldy, int64_t rows, int32_t H, float* partial,
                                   float* loss, void* stream) {
    DLE_CHECK_ARG(x && y && partial && loss && rows > 0 && H > 0 && H % 8 == 0 && ldx >= H && ldy >= H && ldx % 8 == 0 && ldy % 8 == 0);
    DLE_CHECK_ARG(aligned16(x) && aligned16(y));
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const long long nb = (rows + COS_ROWS_PER_BLOCK - 1) / COS_ROWS_PER_BLOCK;
    cosine_rows_fwd_kernel<<<(unsigned)nb, COS_THREADS, 0, st>>>(reinterpret_cast<const bf16*>(x), ldx, reinterpret_cast<const bf16*>(y),
                                                                 ldy, rows, H, partial);
    DLE_LAUNCH_CHECK();
    sum_partials_kernel<<<1, FIN_THREADS, 0, st>>>(partial, nb, 1.0f / (float)rows, loss);
    DLE_LAUNCH_CHECK();
    return DLE_OK;
}

extern "C" int dle_cosine_rows_bwd(const void* x, int64_t ldx, const void* y, int64_t ldy, int64_t rows, int32_t H, const float* grad_scale,
                                   void* dx, int64_t ldd, void* stream) {
    DLE_CHECK_ARG(x && y && grad_scale && dx && rows > 0 && H > 0 && H % 8 == 0 && ldx >= H && ldy >= H && ldd >= H &&
                  ldx % 8 == 0 && ldy % 8 == 0 && ldd % 8 == 0);
    DLE_CHECK_ARG(aligned16(x) && aligned16(y) && aligned16(dx));
    const long long nb = (rows + COS_THREADS / 32 - 1) / (COS_THREADS / 32);
    cosine_rows_bwd_kernel<<<(unsigned)(nb < 4096 ? nb : 4096), COS_THREADS, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
        reinterpret_cast<const bf16*>(x), ldx, reinterpret_cast<const bf16*>(y), ldy, rows, H, grad_scale, 1.0f / (float)rows,
        reinterpret_cast<bf16*>(dx), ldd);
    DLE_LAUNCH_CHECK();
    return DLE_OK;
}

extern "C" int dle_add_rows_bf16(void* dst, int64_t ld_dst, const void* src, int64_t ld_src, int64_t rows, int32_t cols, float* colsum,
                                 void* stream) {
    DLE_CHECK_ARG(dst && src && rows >= 0 && cols > 0 && cols % 2 == 0 && ld_dst >= cols && ld_src >= cols && ld_dst % 2 == 0 &&
                  ld_src % 2 == 0 && (reinterpret_cast<uintptr_t>(dst) & 3) == 0 && (reinterpret_cast<uintptr_t>(src) & 3) == 0);
    if (rows == 0) return DLE_OK;
    const dim3 grid((unsigned)((cols / 2 + 31) / 32), (unsigned)((rows + 8 * ADD_ROWS_PER_THREAD - 1) / (8 * ADD_ROWS_PER_THREAD)));
    add_rows_bf16_kernel<<<grid, dim3(32, 8), 0, reinterpret_cast<cudaStream_t>(stream)>>>(
        reinterpret_cast<bf16*>(dst), ld_dst, reinterpret_cast<const bf16*>(src), ld_src, rows, cols, colsum);
    DLE_LAUNCH_CHECK();
    return DLE_OK;
}
