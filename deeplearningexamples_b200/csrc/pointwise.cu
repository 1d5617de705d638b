// HBM-bound kernels of the BERT encoder path for sm_90a: (bias+)dropout+residual+LayerNorm
// forward/backward, bias+tanh-GELU, embedding gather+LayerNorm, row gathers, column sums, casts.
// All are one-warp-per-row (or 8-element-per-thread) kernels with 128-bit global accesses and
// warp-shuffle reductions; no shared-memory staging is needed because every byte is used once.
//
// replaces (PyTorch/LanguageModeling/BERT/modeling.py): BertSelfOutput/BertOutput :394-398,430-434,
// LinearActivation bias+gelu :121-122,156-160, BertEmbeddings :285-301, index_select :590.
#include "common.cuh"
#include "../../include/dle_b200.h"
#include <stdlib.h>

namespace dle {

constexpr int LN_WARPS = 4;
constexpr int LN_THREADS = LN_WARPS * 32;

static int sm_count() {
    static int sms = 0;
    if (sms == 0) { int dev = 0; cudaGetDevice(&dev); cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev); if (sms <= 0) sms = 132; }
    return sms;
}
static int ln_grid(long long T) {
    long long g = (T + LN_WARPS - 1) / LN_WARPS, cap = (long long)sm_count() * 4;
    return (int)(g < cap ? (g > 0 ? g : 1) : cap);
}

__device__ __forceinline__ void unpack8(const uint4& u, float* f) {
    float2 a = unpack_bf16(u.x), b = unpack_bf16(u.y), c = unpack_bf16(u.z), d = unpack_bf16(u.w);
    f[0] = a.x; f[1] = a.y; f[2] = b.x; f[3] = b.y; f[4] = c.x; f[5] = c.y; f[6] = d.x; f[7] = d.y;
}
__device__ __forceinline__ uint4 pack8(const float* f) {
    return make_uint4(pack_bf16(f[0], f[1]), pack_bf16(f[2], f[3]), pack_bf16(f[4], f[5]), pack_bf16(f[6], f[7]));
}
__device__ __forceinline__ float round_bf16(float x) { return __bfloat162float(__float2bfloat16_rn(x)); }

// LayerNorm statistics of one row held as J*8 values per lane (two-pass in registers)
template <int J> __device__ __forceinline__ void row_stats(const float (&z)[J * 8], int H, float eps, float& mean, float& rstd) {
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < J * 8; ++i) s += z[i];
    mean = warp_sum(s) / (float)H;
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < J * 8; ++i) { float d = z[i] - mean; q += d * d; }
    rstd = 1.0f / sqrtf(warp_sum(q) / (float)H + eps);
}

// ---------------------------------------------------------------------------------------------
// z = dropout(x + bias) + residual ; y = LN(z)
// ---------------------------------------------------------------------------------------------
template <int J>
__global__ void __launch_bounds__(LN_THREADS)
add_ln_fwd_kernel(const bf16* __restrict__ x, const bf16* __restrict__ bias, const bf16* __restrict__ residual,
                  const bf16* __restrict__ gamma, const bf16* __restrict__ beta, bf16* __restrict__ z_out,
                  bf16* __restrict__ y, float* __restrict__ mean_out, float* __restrict__ rstd_out, long long T, float eps,
                  uint32_t thresh, float drop_scale, unsigned long long seed, const unsigned long long* seed_dev, uint32_t stream_id) {
    seed = effective_seed(seed, seed_dev);
    constexpr int H = J * 256;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float gm[J * 8], bt[J * 8], bs[J * 8];
#pragma unroll
    for (int j = 0; j < J; ++j) {
        const int col = j * 256 + lane * 8;
        unpack8(*reinterpret_cast<const uint4*>(gamma + col), gm + j * 8);
        unpack8(*reinterpret_cast<const uint4*>(beta + col), bt + j * 8);
        if (bias) unpack8(*reinterpret_cast<const uint4*>(bias + col), bs + j * 8);
        else {
#pragma unroll
            for (int i = 0; i < 8; ++i) bs[j * 8 + i] = 0.f;
        }
    }
    for (long long row = (long long)blockIdx.x * LN_WARPS + warp; row < T; row += (long long)gridDim.x * LN_WARPS) {
        float z[J * 8];
#pragma unroll
        for (int j = 0; j < J; ++j) {
            const int col = j * 256 + lane * 8;
            unpack8(ld_global_nc_v4(x + row * H + col), z + j * 8);
#pragma unroll
            for (int i = 0; i < 8; ++i) z[j * 8 + i] += bs[j * 8 + i];
            if (thresh != 0u) {
                const uint32_t keep = dropout_keep8(seed, stream_id, (unsigned long long)(row * H + col) >> 5, (col & 31) >> 3, thresh);
#pragma unroll
                for (int i = 0; i < 8; ++i) z[j * 8 + i] = ((keep >> i) & 1u) ? z[j * 8 + i] * drop_scale : 0.f;
            }
            if (residual) {
                float r[8];
                unpack8(ld_global_nc_v4(residual + row * H + col), r);
#pragma unroll
                for (int i = 0; i < 8; ++i) z[j * 8 + i] += r[i];
            }
            if (z_out) {
                // statistics are taken on the bf16 value backward will re-read
#pragma unroll
                for (int i = 0; i < 8; ++i) z[j * 8 + i] = round_bf16(z[j * 8 + i]);
                *reinterpret_cast<uint4*>(z_out + row * H + col) = pack8(z + j * 8);
            }
        }
        float mean, rstd;
        row_stats<J>(z, H, eps, mean, rstd);
        if (lane == 0) { mean_out[row] = mean; rstd_out[row] = rstd; }
#pragma unroll
        for (int j = 0; j < J; ++j) {
            float o[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) o[i] = (z[j * 8 + i] - mean) * rstd * gm[j * 8 + i] + bt[j * 8 + i];
            *reinterpret_cast<uint4*>(y + row * H + j * 256 + lane * 8) = pack8(o);
        }
    }
}

// ---------------------------------------------------------------------------------------------
// LayerNorm backward (+ dropout backward) with fused column partials
// ---------------------------------------------------------------------------------------------
template <int J>
__global__ void __launch_bounds__(LN_THREADS)
add_ln_bwd_kernel(const bf16* __restrict__ dy, const bf16* __restrict__ z, const float* __restrict__ mean_in,
                  const float* __restrict__ rstd_in, const bf16* __restrict__ gamma, bf16* __restrict__ dz_out,
                  bf16* __restrict__ dx_out, float* __restrict__ part_dgamma, float* __restrict__ part_dbeta,
                  float* __restrict__ part_dbias, long long T, uint32_t thresh, float drop_scale,
                  unsigned long long seed, const unsigned long long* seed_dev, uint32_t stream_id) {
    seed = effective_seed(seed, seed_dev);
    constexpr int H = J * 256;
    __shared__ float red[LN_WARPS][H];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float gm[J * 8], ag[J * 8], ab[J * 8], ax[J * 8];
#pragma unroll
    for (int j = 0; j < J; ++j) unpack8(*reinterpret_cast<const uint4*>(gamma + j * 256 + lane * 8), gm + j * 8);
#pragma unroll
    for (int i = 0; i < J * 8; ++i) { ag[i] = 0.f; ab[i] = 0.f; ax[i] = 0.f; }
    const float invH = 1.0f / (float)H;
    for (long long row = (long long)blockIdx.x * LN_WARPS + warp; row < T; row += (long long)gridDim.x * LN_WARPS) {
        const float mean = mean_in[row], rstd = rstd_in[row];
        float g[J * 8], xh[J * 8];
        float s1 = 0.f, s2 = 0.f;
#pragma unroll
        for (int j = 0; j < J; ++j) {
            const int col = j * 256 + lane * 8;
            float d[8], zz[8];
            unpack8(ld_global_nc_v4(dy + row * H + col), d);
            unpack8(ld_global_nc_v4(z + row * H + col), zz);
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const float xhat = (zz[i] - mean) * rstd;
                xh[j * 8 + i] = xhat;
                ag[j * 8 + i] += d[i] * xhat;
                ab[j * 8 + i] += d[i];
                const float gg = d[i] * gm[j * 8 + i];
                g[j * 8 + i] = gg;
                s1 += gg; s2 += gg * xhat;
            }
        }
        s1 = warp_sum(s1) * invH; s2 = warp_sum(s2) * invH;
#pragma unroll
        for (int j = 0; j < J; ++j) {
            const int col = j * 256 + lane * 8;
            float dzv[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) dzv[i] = rstd * (g[j * 8 + i] - s1 - xh[j * 8 + i] * s2);
            if (dz_out) *reinterpret_cast<uint4*>(dz_out + row * H + col) = pack8(dzv);
            if (thresh != 0u) {
                const uint32_t keep = dropout_keep8(seed, stream_id, (unsigned long long)(row * H + col) >> 5, (col & 31) >> 3, thresh);
#pragma unroll
                for (int i = 0; i < 8; ++i) dzv[i] = ((keep >> i) & 1u) ? dzv[i] * drop_scale : 0.f;
                if (dx_out) *reinterpret_cast<uint4*>(dx_out + row * H + col) = pack8(dzv);
            }
#pragma unroll
            for (int i = 0; i < 8; ++i) ax[j * 8 + i] += round_bf16(dzv[i]);   // bias grad sums what the GEMM will read
        }
    }
    // cross-warp reduction of the three column partials, one after the other through `red`
    float* outs[3] = {part_dgamma, part_dbeta, part_dbias};
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        if (outs[k] == nullptr) continue;
        __syncthreads();
#pragma unroll
        for (int j = 0; j < J; ++j)
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const float v = (k == 0) ? ag[j * 8 + i] : (k == 1 ? ab[j * 8 + i] : ax[j * 8 + i]);
                red[warp][j * 256 + lane * 8 + i] = v;
            }
        __syncthreads();
        for (int c = threadIdx.x; c < H; c += LN_THREADS) {
            float s = 0.f;
#pragma unroll
            for (int w = 0; w < LN_WARPS; ++w) s += red[w][c];
            outs[k][(long long)blockIdx.x * H + c] = s;
        }
    }
}

// ---------------------------------------------------------------------------------------------
// Two-warps-per-row variants (H % 512 == 0).  The one-warp-per-row kernels above keep 3 x 32 column accumulators + 32 gammas
// per lane (255 registers at H = 1024 => 8 resident warps per SM, ~50 % of HBM peak); with 64 lanes per row each lane owns
// 16 columns, registers halve and occupancy doubles.  Row statistics cross the two warps through a double-buffered smem slot
// and a 64-thread named barrier.
// ---------------------------------------------------------------------------------------------
constexpr int LN2_ROWS = 4;                       // row groups per CTA
constexpr int LN2_THREADS = LN2_ROWS * 64;
constexpr int LN2_DEPTH = 3;                      // rows per warp pair in flight (cp.async prefetch ring)

__device__ __forceinline__ void pair_bar(int rg) { asm volatile("bar.sync %0, 64;" ::"r"(rg + 1) : "memory"); }

template <int J2>   // H = J2 * 512
__global__ void __launch_bounds__(LN2_THREADS)
add_ln_fwd2_kernel(const bf16* __restrict__ x, const bf16* __restrict__ bias, const bf16* __restrict__ residual,
                   const bf16* __restrict__ gamma, const bf16* __restrict__ beta, bf16* __restrict__ z_out,
                   bf16* __restrict__ y, float* __restrict__ mean_out, float* __restrict__ rstd_out, long long T, float eps,
                   uint32_t thresh, float drop_scale, unsigned long long seed, const unsigned long long* seed_dev, uint32_t stream_id) {
    seed = effective_seed(seed, seed_dev);
    constexpr int H = J2 * 512;
    __shared__ float ex[2][LN2_ROWS][2][2];        // [parity][row group][warp of the pair][slot]
    const int t64 = threadIdx.x & 63, rg = threadIdx.x >> 6, wp = (threadIdx.x >> 5) & 1, lane = threadIdx.x & 31;
    uint4 gm[J2], bt[J2], bs[J2];
#pragma unroll
    for (int j = 0; j < J2; ++j) {
        const int col = j * 512 + t64 * 8;
        gm[j] = *reinterpret_cast<const uint4*>(gamma + col);
        bt[j] = *reinterpret_cast<const uint4*>(beta + col);
        bs[j] = bias ? *reinterpret_cast<const uint4*>(bias + col) : make_uint4(0u, 0u, 0u, 0u);
    }
    int par = 0;
    // Prefetch ring: every thread copies ITS OWN 16-byte pieces of the next LN2_DEPTH rows into a private shared-memory slot with
    // cp.async (no registers, no barrier: a thread only ever reads back what it copied), so LN2_DEPTH rows per warp pair are in
    // flight.  Round 1 had one row in flight (2.6 TB/s: 16 resident warps x 32 B per lane do not cover HBM's latency-bandwidth
    // product), a register double buffer reached 4.5 TB/s.
    __shared__ uint4 ring[LN2_DEPTH][J2][LN2_THREADS];
    const long long stride = (long long)gridDim.x * LN2_ROWS;
    long long row = (long long)blockIdx.x * LN2_ROWS + rg;
    auto prefetch = [&](int slot, long long r_) {
        if (r_ < T) {
#pragma unroll
            for (int j = 0; j < J2; ++j) cp_async16(smem_u32(&ring[slot][j][threadIdx.x]), x + r_ * H + j * 512 + t64 * 8);
        }
        cp_async_commit();
    };
#pragma unroll
    for (int d = 0; d < LN2_DEPTH; ++d) prefetch(d, row + d * stride);
    int slot = 0;
    for (; row < T; row += stride, par ^= 1) {
        float z[J2 * 8];
        float s = 0.f;
        uint4 cur[J2];
        cp_async_wait<LN2_DEPTH - 1>();
#pragma unroll
        for (int j = 0; j < J2; ++j) cur[j] = lds_u4(smem_u32(&ring[slot][j][threadIdx.x]));
        prefetch(slot, row + LN2_DEPTH * stride);
        slot = (slot + 1 == LN2_DEPTH) ? 0 : slot + 1;
#pragma unroll
        for (int j = 0; j < J2; ++j) {
            const int col = j * 512 + t64 * 8;
            float b[8];
            unpack8(cur[j], z + j * 8);
            unpack8(bs[j], b);
#pragma unroll
            for (int i = 0; i < 8; ++i) z[j * 8 + i] += b[i];
            if (thresh != 0u) {
                const uint32_t keep = dropout_keep8(seed, stream_id, (unsigned long long)(row * H + col) >> 5, (col & 31) >> 3, thresh);
#pragma unroll
                for (int i = 0; i < 8; ++i) z[j * 8 + i] = ((keep >> i) & 1u) ? z[j * 8 + i] * drop_scale : 0.f;
            }
            if (residual) {
                float r[8];
                unpack8(ld_global_nc_v4(residual + row * H + col), r);
#pragma unroll
                for (int i = 0; i < 8; ++i) z[j * 8 + i] += r[i];
            }
            if (z_out) {
#pragma unroll
                for (int i = 0; i < 8; ++i) z[j * 8 + i] = round_bf16(z[j * 8 + i]);
                *reinterpret_cast<uint4*>(z_out + row * H + col) = pack8(z + j * 8);
            }
#pragma unroll
            for (int i = 0; i < 8; ++i) s += z[j * 8 + i];
        }
        s = warp_sum(s);
        if (lane == 0) ex[par][rg][wp][0] = s;
        pair_bar(rg);
        const float mean = (ex[par][rg][0][0] + ex[par][rg][1][0]) / (float)H;
        float q = 0.f;
#pragma unroll
        for (int i = 0; i < J2 * 8; ++i) { const float d = z[i] - mean; q += d * d; }
        q = warp_sum(q);
        if (lane == 0) ex[par][rg][wp][1] = q;
        pair_bar(rg);
        const float rstd = 1.0f / sqrtf((ex[par][rg][0][1] + ex[par][rg][1][1]) / (float)H + eps);
        if (t64 == 0) { mean_out[row] = mean; rstd_out[row] = rstd; }
#pragma unroll
        for (int j = 0; j < J2; ++j) {
            float g[8], b[8], o[8];
            unpack8(gm[j], g); unpack8(bt[j], b);
#pragma unroll
            for (int i = 0; i < 8; ++i) o[i] = (z[j * 8 + i] - mean) * rstd * g[i] + b[i];
            *reinterpret_cast<uint4*>(y + row * H + j * 512 + t64 * 8) = pack8(o);
        }
    }
}

template <int J2>
__global__ void __launch_bounds__(LN2_THREADS, J2 == 1 ? 4 : 2)
add_ln_bwd2_kernel(const bf16* __restrict__ dy, const bf16* __restrict__ z, const float* __restrict__ mean_in,
                   const float* __restrict__ rstd_in, const bf16* __restrict__ gamma, bf16* __restrict__ dz_out,
                   bf16* __restrict__ dx_out, float* __restrict__ part_dgamma, float* __restrict__ part_dbeta,
                   float* __restrict__ part_dbias, long long T, uint32_t thresh, float drop_scale,
                   unsigned long long seed, const unsigned long long* seed_dev, uint32_t stream_id) {
    seed = effective_seed(seed, seed_dev);
    constexpr int H = J2 * 512;
    __shared__ float ex[2][LN2_ROWS][2][2];
    extern __shared__ __align__(16) uint8_t ln_smem[];          // max(prefetch ring, column-reduction buffer)
    float (*red)[H] = reinterpret_cast<float (*)[H]>(ln_smem);
    const int t64 = threadIdx.x & 63, rg = threadIdx.x >> 6, wp = (threadIdx.x >> 5) & 1, lane = threadIdx.x & 31;
    uint4 gm[J2];
    float ag[J2 * 8], ab[J2 * 8], ax[J2 * 8];
#pragma unroll
    for (int j = 0; j < J2; ++j) gm[j] = *reinterpret_cast<const uint4*>(gamma + j * 512 + t64 * 8);
#pragma unroll
    for (int i = 0; i < J2 * 8; ++i) { ag[i] = 0.f; ab[i] = 0.f; ax[i] = 0.f; }
    const float invH = 1.0f / (float)H;
    int par = 0;
    // cp.async prefetch ring (see add_ln_fwd2_kernel): LN2_DEPTH rows of dy and z per warp pair in flight, no staging registers.  The
    // ring aliases the column-reduction buffer `red`, which is only used after the row loop.
    uint4 (*ring)[2 * J2][LN2_THREADS] = reinterpret_cast<uint4 (*)[2 * J2][LN2_THREADS]>(ln_smem);
    const long long stride = (long long)gridDim.x * LN2_ROWS;
    long long row = (long long)blockIdx.x * LN2_ROWS + rg;
    auto prefetch = [&](int slot, long long r_) {
        if (r_ < T) {
#pragma unroll
            for (int j = 0; j < J2; ++j) {
                cp_async16(smem_u32(&ring[slot][j][threadIdx.x]), dy + r_ * H + j * 512 + t64 * 8);
                cp_async16(smem_u32(&ring[slot][J2 + j][threadIdx.x]), z + r_ * H + j * 512 + t64 * 8);
            }
        }
        cp_async_commit();
    };
#pragma unroll
    for (int d = 0; d < LN2_DEPTH; ++d) prefetch(d, row + d * stride);
    float nmean = 0.f, nrstd = 0.f;
    if (row < T) { nmean = mean_in[row]; nrstd = rstd_in[row]; }
    int slot = 0;
    for (; row < T; row += stride, par ^= 1) {
        const float mean = nmean, rstd = nrstd;
        uint4 cdy[J2], cz[J2];
        cp_async_wait<LN2_DEPTH - 1>();
#pragma unroll
        for (int j = 0; j < J2; ++j) {
            cdy[j] = lds_u4(smem_u32(&ring[slot][j][threadIdx.x]));
            cz[j] = lds_u4(smem_u32(&ring[slot][J2 + j][threadIdx.x]));
        }
        prefetch(slot, row + LN2_DEPTH * stride);
        slot = (slot + 1 == LN2_DEPTH) ? 0 : slot + 1;
        if (row + stride < T) { nmean = mean_in[row + stride]; nrstd = rstd_in[row + stride]; }
        float g[J2 * 8], xh[J2 * 8];
        float s1 = 0.f, s2 = 0.f;
#pragma unroll
        for (int j = 0; j < J2; ++j) {
            float d[8], zz[8], gg[8];
            unpack8(cdy[j], d);
            unpack8(cz[j], zz);
            unpack8(gm[j], gg);
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const float xhat = (zz[i] - mean) * rstd;
                xh[j * 8 + i] = xhat;
                ag[j * 8 + i] += d[i] * xhat;
                ab[j * 8 + i] += d[i];
                const float t = d[i] * gg[i];
                g[j * 8 + i] = t;
                s1 += t; s2 += t * xhat;
            }
        }
        s1 = warp_sum(s1); s2 = warp_sum(s2);
        if (lane == 0) { ex[par][rg][wp][0] = s1; ex[par][rg][wp][1] = s2; }
        pair_bar(rg);
        s1 = (ex[par][rg][0][0] + ex[par][rg][1][0]) * invH;
        s2 = (ex[par][rg][0][1] + ex[par][rg][1][1]) * invH;
#pragma unroll
        for (int j = 0; j < J2; ++j) {
            const int col = j * 512 + t64 * 8;
            float dzv[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) dzv[i] = rstd * (g[j * 8 + i] - s1 - xh[j * 8 + i] * s2);
            if (dz_out) *reinterpret_cast<uint4*>(dz_out + row * H + col) = pack8(dzv);
            if (thresh != 0u) {
                const uint32_t keep = dropout_keep8(seed, stream_id, (unsigned long long)(row * H + col) >> 5, (col & 31) >> 3, thresh);
#pragma unroll
                for (int i = 0; i < 8; ++i) dzv[i] = ((keep >> i) & 1u) ? dzv[i] * drop_scale : 0.f;
                if (dx_out) *reinterpret_cast<uint4*>(dx_out + row * H + col) = pack8(dzv);
            }
#pragma unroll
            for (int i = 0; i < 8; ++i) ax[j * 8 + i] += round_bf16(dzv[i]);
        }
    }
    cp_async_wait<0>();
    float* outs[3] = {part_dgamma, part_dbeta, part_dbias};
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        if (outs[k] == nullptr) continue;
        __syncthreads();
#pragma unroll
        for (int j = 0; j < J2; ++j)
#pragma unroll
            for (int i = 0; i < 8; ++i) red[rg][j * 512 + t64 * 8 + i] = (k == 0) ? ag[j * 8 + i] : (k == 1 ? ab[j * 8 + i] : ax[j * 8 + i]);
        __syncthreads();
        for (int c = threadIdx.x; c < H; c += LN2_THREADS) {
            float t = 0.f;
#pragma unroll
            for (int w = 0; w < LN2_ROWS; ++w) t += red[w][c];
            outs[k][(long long)blockIdx.x * H + c] = t;
        }
    }
}
// DLE_LN_ONE_WARP=1 selects the one-warp-per-row kernels (A/B measurements)
static bool ln_force_one_warp() { const char* e = getenv("DLE_LN_ONE_WARP"); return e && e[0] == '1'; }
static int ln2_bwd_smem(int j2) {                 // bytes: the larger of the prefetch ring and the [LN2_ROWS][H] fp32 reduction buffer
    const int ring = LN2_DEPTH * 2 * j2 * LN2_THREADS * 16, red = LN2_ROWS * j2 * 512 * 4;
    return ring > red ? ring : red;
}
template <int J2> static int ln2_bwd_attr() {       // > 48 KB of shared memory per CTA needs the opt-in attribute (per device)
    static bool done[64] = {};
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return DLE_ERR_CUDA;
    if (!done[dev]) {
        if (cudaFuncSetAttribute(add_ln_bwd2_kernel<J2>, cudaFuncAttributeMaxDynamicSharedMemorySize, ln2_bwd_smem(J2)) != cudaSuccess) return DLE_ERR_CUDA;
        done[dev] = true;
    }
    return DLE_OK;
}
static int ln2_grid(long long T) {
    long long g = (T + LN2_ROWS - 1) / LN2_ROWS, cap = (long long)sm_count() * 4;
    return (int)(g < cap ? (g > 0 ? g : 1) : cap);
}

// out[a][n] = sum_p part[a][p][n]   (grid: (ceil(N/32), n_arrays); 16 warps stride over the partial rows, each
// warp reading 128 contiguous bytes per row; cross-warp reduction through shared memory)
constexpr int CF_WARPS = 16;
__global__ void __launch_bounds__(CF_WARPS * 32)
colsum_finalize_kernel(const float* __restrict__ part, int n_part, int N, void* out, int out_dtype, int accumulate) {
    __shared__ float red[CF_WARPS][33];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int n = blockIdx.x * 32 + lane;
    const float* src = part + (long long)blockIdx.y * n_part * N;
    float s = 0.f;
    if (n < N) {
        int p = warp;
        for (; p + 3 * CF_WARPS < n_part; p += 4 * CF_WARPS) {
            const float a = src[(long long)p * N + n], b = src[(long long)(p + CF_WARPS) * N + n];
            const float c = src[(long long)(p + 2 * CF_WARPS) * N + n], d = src[(long long)(p + 3 * CF_WARPS) * N + n];
            s += (a + b) + (c + d);
        }
        for (; p < n_part; p += CF_WARPS) s += src[(long long)p * N + n];
    }
    red[warp][lane] = s;
    __syncthreads();
    if (warp == 0 && n < N) {
        float t = 0.f;
#pragma unroll
        for (int w = 0; w < CF_WARPS; ++w) t += red[w][lane];
        const long long o_idx = (long long)blockIdx.y * N + n;
        if (out_dtype == DLE_DTYPE_F32) {
            float* o = reinterpret_cast<float*>(out);
            o[o_idx] = accumulate ? o[o_idx] + t : t;
        } else {
            bf16* o = reinterpret_cast<bf16*>(out);
            o[o_idx] = __float2bfloat16_rn(accumulate ? __bfloat162float(o[o_idx]) + t : t);
        }
    }
}

// column sums of a bf16 [T, N] matrix: grid (col blocks of 256, row slabs), 8 warps per CTA
constexpr int CS_WARPS = 8;
__global__ void __launch_bounds__(CS_WARPS * 32)
colsum_bf16_kernel(const bf16* __restrict__ x, long long T, int N, long long ldx, float* __restrict__ part, int rows_per_slab) {
    __shared__ float red[CS_WARPS][256];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int col = blockIdx.x * 256 + lane * 8;
    const long long r0 = (long long)blockIdx.y * rows_per_slab;
    const long long r1 = min(T, r0 + rows_per_slab);
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    if (col < N) {
        for (long long r = r0 + warp; r < r1; r += CS_WARPS) {
            float f[8];
            unpack8(ld_global_nc_v4(x + r * ldx + col), f);
#pragma unroll
            for (int i = 0; i < 8; ++i) acc[i] += f[i];
        }
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) red[warp][lane * 8 + i] = acc[i];
    __syncthreads();
    const int c = threadIdx.x;
    if (c < 256 && blockIdx.x * 256 + c < N) {
        float s = 0.f;
#pragma unroll
        for (int w = 0; w < CS_WARPS; ++w) s += red[w][c];
        part[(long long)blockIdx.y * N + blockIdx.x * 256 + c] = s;
    }
}

// ---------------------------------------------------------------------------------------------
// bias + tanh-GELU standalone
// ---------------------------------------------------------------------------------------------
__global__ void bias_gelu_fwd_kernel(const bf16* __restrict__ x, const bf16* __restrict__ bias, bf16* __restrict__ u_out,
                                     bf16* __restrict__ y, long long T, int N) {
    const long long nvec = T * N / 8;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += (long long)gridDim.x * blockDim.x) {
        float f[8], b[8];
        unpack8(ld_global_nc_v4(x + i * 8), f);
        if (bias) {
            unpack8(*reinterpret_cast<const uint4*>(bias + (i * 8) % N), b);
#pragma unroll
            for (int k = 0; k < 8; ++k) f[k] = round_bf16(f[k] + b[k]);
        }
        if (u_out) *reinterpret_cast<uint4*>(u_out + i * 8) = pack8(f);
#pragma unroll
        for (int k = 0; k < 8; ++k) f[k] = gelu_tanh(f[k]);
        *reinterpret_cast<uint4*>(y + i * 8) = pack8(f);
    }
}
__global__ void bias_gelu_bwd_kernel(const bf16* __restrict__ dy, const bf16* __restrict__ u, bf16* __restrict__ du, long long nvec) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += (long long)gridDim.x * blockDim.x) {
        float d[8], uu[8];
        unpack8(ld_global_nc_v4(dy + i * 8), d);
        unpack8(ld_global_nc_v4(u + i * 8), uu);
#pragma unroll
        for (int k = 0; k < 8; ++k) d[k] *= gelu_tanh_grad(uu[k]);
        *reinterpret_cast<uint4*>(du + i * 8) = pack8(d);
    }
}

// ---------------------------------------------------------------------------------------------
// embeddings: z = word[id] + pos[s] + type[tt] ; y = dropout(LN(z))
// ---------------------------------------------------------------------------------------------
template <int J>
__global__ void __launch_bounds__(LN_THREADS)
embed_ln_fwd_kernel(const long long* __restrict__ ids, const long long* __restrict__ tts, const bf16* __restrict__ word,
                    const bf16* __restrict__ pos, const bf16* __restrict__ type, const bf16* __restrict__ gamma,
                    const bf16* __restrict__ beta, bf16* __restrict__ z_out, bf16* __restrict__ y, float* __restrict__ mean_out,
                    float* __restrict__ rstd_out, int B, int S, int V, int P, int NT, float eps, uint32_t thresh,
                    float drop_scale, unsigned long long seed, const unsigned long long* seed_dev, uint32_t stream_id, int* err_flag,
                    const long long* __restrict__ pos_ids) {
    seed = effective_seed(seed, seed_dev);
    constexpr int H = J * 256;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const long long T = (long long)B * S;
    float gm[J * 8], bt[J * 8];
#pragma unroll
    for (int j = 0; j < J; ++j) {
        unpack8(*reinterpret_cast<const uint4*>(gamma + j * 256 + lane * 8), gm + j * 8);
        unpack8(*reinterpret_cast<const uint4*>(beta + j * 256 + lane * 8), bt + j * 8);
    }
    for (long long row = (long long)blockIdx.x * LN_WARPS + warp; row < T; row += (long long)gridDim.x * LN_WARPS) {
        long long id = ids[row], tt = tts[row];
        long long sp = pos_ids ? pos_ids[row] : row % S;         // explicit positions restart per packed sample
        if (id < 0 || id >= V || tt < 0 || tt >= NT || sp < 0 || sp >= P) {
            if (err_flag && lane == 0) atomicExch(err_flag, 1);
            id = 0; tt = 0; sp = 0;
        }
        const int s = (int)sp;
        float z[J * 8];
#pragma unroll
        for (int j = 0; j < J; ++j) {
            const int col = j * 256 + lane * 8;
            float a[8], b[8], c[8];
            unpack8(ld_global_nc_v4(word + id * H + col), a);
            unpack8(ld_global_nc_v4(pos + (long long)s * H + col), b);
            unpack8(ld_global_nc_v4(type + tt * H + col), c);
#pragma unroll
            for (int i = 0; i < 8; ++i) z[j * 8 + i] = round_bf16(a[i] + b[i] + c[i]);
            if (z_out) *reinterpret_cast<uint4*>(z_out + row * H + col) = pack8(z + j * 8);
        }
        float mean, rstd;
        row_stats<J>(z, H, eps, mean, rstd);
        if (lane == 0) { mean_out[row] = mean; rstd_out[row] = rstd; }
#pragma unroll
        for (int j = 0; j < J; ++j) {
            const int col = j * 256 + lane * 8;
            float o[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) o[i] = (z[j * 8 + i] - mean) * rstd * gm[j * 8 + i] + bt[j * 8 + i];
            if (thresh != 0u) {
                const uint32_t keep = dropout_keep8(seed, stream_id, (unsigned long long)(row * H + col) >> 5, (col & 31) >> 3, thresh);
#pragma unroll
                for (int i = 0; i < 8; ++i) o[i] = ((keep >> i) & 1u) ? o[i] * drop_scale : 0.f;
            }
            *reinterpret_cast<uint4*>(y + row * H + col) = pack8(o);
        }
    }
}

template <int J>
__global__ void __launch_bounds__(LN_THREADS)
embed_ln_bwd_kernel(const bf16* __restrict__ dy, const bf16* __restrict__ z, const float* __restrict__ mean_in,
                    const float* __restrict__ rstd_in, const bf16* __restrict__ gamma, const long long* __restrict__ ids,
                    const long long* __restrict__ tts, float* __restrict__ dword, float* __restrict__ dpos,
                    float* __restrict__ dtype_tab, float* __restrict__ part_dgamma, float* __restrict__ part_dbeta,
                    int B, int S, uint32_t thresh, float drop_scale, unsigned long long seed, const unsigned long long* seed_dev, uint32_t stream_id,
                    const long long* __restrict__ pos_ids) {
    seed = effective_seed(seed, seed_dev);
    constexpr int H = J * 256;
    __shared__ float red[LN_WARPS][H];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const long long T = (long long)B * S;
    float gm[J * 8], ag[J * 8], ab[J * 8];
#pragma unroll
    for (int j = 0; j < J; ++j) unpack8(*reinterpret_cast<const uint4*>(gamma + j * 256 + lane * 8), gm + j * 8);
#pragma unroll
    for (int i = 0; i < J * 8; ++i) { ag[i] = 0.f; ab[i] = 0.f; }
    const float invH = 1.0f / (float)H;
    for (long long row = (long long)blockIdx.x * LN_WARPS + warp; row < T; row += (long long)gridDim.x * LN_WARPS) {
        const float mean = mean_in[row], rstd = rstd_in[row];
        float g[J * 8], xh[J * 8];
        float s1 = 0.f, s2 = 0.f;
#pragma unroll
        for (int j = 0; j < J; ++j) {
            const int col = j * 256 + lane * 8;
            float d[8], zz[8];
            unpack8(ld_global_nc_v4(dy + row * H + col), d);
            unpack8(ld_global_nc_v4(z + row * H + col), zz);
            if (thresh != 0u) {
                const uint32_t keep = dropout_keep8(seed, stream_id, (unsigned long long)(row * H + col) >> 5, (col & 31) >> 3, thresh);
#pragma unroll
                for (int i = 0; i < 8; ++i) d[i] = ((keep >> i) & 1u) ? d[i] * drop_scale : 0.f;
            }
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const float xhat = (zz[i] - mean) * rstd;
                xh[j * 8 + i] = xhat;
                ag[j * 8 + i] += d[i] * xhat;
                ab[j * 8 + i] += d[i];
                const float gg = d[i] * gm[j * 8 + i];
                g[j * 8 + i] = gg;
                s1 += gg; s2 += gg * xhat;
            }
        }
        s1 = warp_sum(s1) * invH; s2 = warp_sum(s2) * invH;
        const long long id = ids[row], tt = tts[row];
        const int s = (int)(pos_ids ? pos_ids[row] : row % S);
#pragma unroll
        for (int j = 0; j < J; ++j) {
            const int col = j * 256 + lane * 8;
            float dzv[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) dzv[i] = rstd * (g[j * 8 + i] - s1 - xh[j * 8 + i] * s2);
            red_add_v4_f32(dword + id * H + col, dzv[0], dzv[1], dzv[2], dzv[3]);
            red_add_v4_f32(dword + id * H + col + 4, dzv[4], dzv[5], dzv[6], dzv[7]);
            red_add_v4_f32(dpos + (long long)s * H + col, dzv[0], dzv[1], dzv[2], dzv[3]);
            red_add_v4_f32(dpos + (long long)s * H + col + 4, dzv[4], dzv[5], dzv[6], dzv[7]);
            red_add_v4_f32(dtype_tab + tt * H + col, dzv[0], dzv[1], dzv[2], dzv[3]);
            red_add_v4_f32(dtype_tab + tt * H + col + 4, dzv[4], dzv[5], dzv[6], dzv[7]);
        }
    }
    float* outs[2] = {part_dgamma, part_dbeta};
#pragma unroll
    for (int k = 0; k < 2; ++k) {
        __syncthreads();
#pragma unroll
        for (int j = 0; j < J; ++j)
#pragma unroll
            for (int i = 0; i < 8; ++i) red[warp][j * 256 + lane * 8 + i] = (k == 0) ? ag[j * 8 + i] : ab[j * 8 + i];
        __syncthreads();
        for (int c = threadIdx.x; c < H; c += LN_THREADS) {
            float s = 0.f;
#pragma unroll
            for (int w = 0; w < LN_WARPS; ++w) s += red[w][c];
            outs[k][(long long)blockIdx.x * H + c] = s;
        }
    }
}

// ---------------------------------------------------------------------------------------------
// row gather / scatter (bit-exact copies), casts
// ---------------------------------------------------------------------------------------------
__global__ void gather_rows_kernel(const bf16* __restrict__ x, const long long* __restrict__ idx, bf16* __restrict__ out,
                                   long long n_idx, int H, long long n_rows, int* err_flag) {
    const int vec_per_row = H / 8;
    const long long total = n_idx * vec_per_row;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const long long r = i / vec_per_row; const int c = (int)(i - r * vec_per_row);
        long long src = idx[r];
        if (src == -1) {                                          // padding slot (static-size index lists): zero row, not an error
            *reinterpret_cast<uint4*>(out + r * H + c * 8) = make_uint4(0u, 0u, 0u, 0u);
            continue;
        }
        if (src < 0 || src >= n_rows) { if (err_flag) atomicExch(err_flag, 1); src = 0; }
        *reinterpret_cast<uint4*>(out + r * H + c * 8) = ld_global_nc_v4(x + src * H + c * 8);
    }
}
__global__ void scatter_rows_kernel(const bf16* __restrict__ dy, const long long* __restrict__ idx, bf16* __restrict__ dx,
                                    long long n_idx, int H, long long n_rows) {
    const int vec_per_row = H / 8;
    const long long total = n_idx * vec_per_row;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const long long r = i / vec_per_row; const int c = (int)(i - r * vec_per_row);
        const long long dst = idx[r];
        if (dst < 0 || dst >= n_rows) continue;
        *reinterpret_cast<uint4*>(dx + dst * H + c * 8) = ld_global_nc_v4(dy + r * H + c * 8);
    }
}
// ---------------------------------------------------------------------------------------------
// segment table of a packed batch: mask[b, s] = sample number j (1..k, contiguous, increasing), 0 on the row's padding tail
// ---------------------------------------------------------------------------------------------
constexpr int SEG_WARPS = 4;

// one warp per row, two passes over the row in 32-token chunks: (1) validate and find the row's real-token count n and sample count m,
// (2) write positions, segment starts and [CLS] rows.  A malformed row is written as if its mask were all 0 (one tail segment).
__global__ void __launch_bounds__(SEG_WARPS * 32)
segment_table_kernel(const long long* __restrict__ mask, int B, int S, int k, int* __restrict__ cu_seqlens,
                     long long* __restrict__ position_ids, long long* __restrict__ cls_index, int* err_flag) {
    const int lane = threadIdx.x & 31;
    const int b = blockIdx.x * SEG_WARPS + (threadIdx.x >> 5);
    if (b >= B) return;
    const long long* m_row = mask + (long long)b * S;
    const long long row0 = (long long)b * S;
    // pass 1: every token must satisfy 0 <= v <= k and v == 0 || (s == 0 ? v == 1 : prev != 0 && (v == prev || v == prev + 1))
    bool bad = false;
    int n = 0, m = 0;
    long long carry = 0;                                     // value of the token before this chunk (0 before the row)
    for (int base = 0; base < S; base += 32) {
        const int s = base + lane;
        const long long v = s < S ? m_row[s] : 0;
        long long prev = __shfl_up_sync(0xffffffffu, v, 1);
        if (lane == 0) prev = carry;
        if (s < S) {
            const bool ok = v >= 0 && v <= k && (v == 0 || (s == 0 ? v == 1 : prev != 0 && (v == prev || v == prev + 1)));
            bad |= !ok;
            if (v != 0) { ++n; m = max(m, (int)min(v, (long long)k)); }
        }
        carry = __shfl_sync(0xffffffffu, v, 31);
    }
    bad = __any_sync(0xffffffffu, bad);
    n = __reduce_add_sync(0xffffffffu, n);
    m = __reduce_max_sync(0xffffffffu, m);
    if (bad) {
        if (err_flag && lane == 0) atomicExch(err_flag, 1);
        n = 0; m = 0;
    }
    int* cu = cu_seqlens + (long long)b * (k + 1);
    // pass 2: a segment starts where the value changes (and at s == 0); position = s - start of the token's segment
    int seg = 0;                                             // start of the segment the previous chunk ended in
    carry = 0;
    for (int base = 0; base < S; base += 32) {
        const int s = base + lane;
        const long long v = (s < S && !bad) ? m_row[s] : 0;
        long long prev = __shfl_up_sync(0xffffffffu, v, 1);
        if (lane == 0) prev = carry;
        const bool start = s < S && (s == 0 || v != prev);
        int st = start ? s : -1;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {                   // inclusive max-scan of segment starts over the chunk
            const int o = __shfl_up_sync(0xffffffffu, st, d);
            if (lane >= d) st = max(st, o);
        }
        st = max(st, seg);
        if (s < S) {
            position_ids[row0 + s] = s - st;
            if (start && v != 0) {                           // sample v starts here (the tail's start is written below)
                cu[v - 1] = (int)(row0 + s);
                cls_index[(long long)b * k + v - 1] = row0 + s;
            }
        }
        seg = __shfl_sync(0xffffffffu, st, 31);
        carry = __shfl_sync(0xffffffffu, v, 31);
    }
    // absent samples are empty segments at the tail's start; the tail is segment k
    for (int j = m + 1 + lane; j <= k + 1; j += 32) {
        cu[j - 1] = (int)(row0 + n);
        if (j <= k) cls_index[(long long)b * k + j - 1] = -1;
    }
    if (b == B - 1 && lane == 0) cu_seqlens[(long long)B * (k + 1)] = (int)((long long)B * S);
}
// ---------------------------------------------------------------------------------------------
// per-sample span logits of a packed batch: the QA head's [B*S, 2] output on the packed grid <-> [B*k, S] start / end rows,
// one per sample slot; slot b*k + j is sequence b*(k+1) + j of the segment table.  Pure moves: bit exact both ways.
// ---------------------------------------------------------------------------------------------
template <typename T>
__global__ void span_logits_unpack_kernel(const T* __restrict__ logits, long long ld, const int* __restrict__ cu_seqlens, int S, int k,
                                          long long n, float fill, T* __restrict__ start_out, T* __restrict__ end_out) {
    const T f = static_cast<T>(fill);
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const long long slot = i / S;
        const int p = (int)(i - slot * S);
        const long long seq = slot / k * (k + 1) + slot % k;
        const int c0 = cu_seqlens[seq];
        T s = f, e = f;
        if (p < cu_seqlens[seq + 1] - c0) {
            const T* row = logits + (long long)(c0 + p) * ld;
            s = row[0];
            e = row[1];
        }
        start_out[i] = s;
        end_out[i] = e;
    }
}
// one thread per grid token: every row of dlogits is written exactly once (tail tokens get 0), so no memset and no atomics
template <typename T>
__global__ void span_logits_pack_grad_kernel(const T* __restrict__ dstart, const T* __restrict__ dend, const int* __restrict__ cu_seqlens,
                                             int S, int k, long long n, T* __restrict__ dlogits, long long ld) {
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < n; t += (long long)gridDim.x * blockDim.x) {
        const long long b = t / S;
        const int* cu = cu_seqlens + b * (k + 1);
        // the row's sequence holding t: the last of its k+1 starts that is <= t (an empty slot starts where the next one does)
        int lo = 0, hi = k;
        while (lo < hi) {
            const int mid = (lo + hi + 1) >> 1;
            if (cu[mid] <= t) lo = mid; else hi = mid - 1;
        }
        T ds = static_cast<T>(0.f), de = static_cast<T>(0.f);
        if (lo < k) {                                          // lo == k: the row's padding tail
            const long long o = (b * k + lo) * S + (t - cu[lo]);
            ds = dstart[o];
            de = dend[o];
        }
        dlogits[t * ld] = ds;
        dlogits[t * ld + 1] = de;
    }
}
// ---------------------------------------------------------------------------------------------
// sequence-classification head: logits[r, l] = sum_c dropout(x)[r, c] * W[l, c] + b[l] (modeling.py:1145-1155), L <= 32 labels,
// too narrow for the GEMM (N % 8).  The dropout keep bit of x[r, c] is that of flat element r*H + c, as at every hidden-dropout site.
// Each row's arithmetic depends on that row alone.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float ld_f32(const float* p) { return *p; }
__device__ __forceinline__ float ld_f32(const bf16* p) { return __bfloat162float(*p); }
__device__ __forceinline__ void st_f32(float* p, float v) { *p = v; }
__device__ __forceinline__ void st_f32(bf16* p, float v) { *p = __float2bfloat16_rn(v); }

// forward: one warp per row, lane owns the 8-column units lane, lane + 32, ...; labels CLS_LC at a time (dropout redrawn per pass);
// lane-order fp32 partial sums, then a butterfly warp sum: a fixed order per row
constexpr int CLS_WARPS = 8, CLS_LC = 4;
template <typename T>
__global__ void __launch_bounds__(CLS_WARPS * 32)
cls_head_fwd_kernel(const bf16* __restrict__ x, long long ldx, const bf16* __restrict__ w, const T* __restrict__ b, int R, int H, int L,
                    uint32_t thresh, float drop_scale, unsigned long long seed, const unsigned long long* seed_dev, uint32_t stream_id,
                    T* __restrict__ logits) {
    seed = effective_seed(seed, seed_dev);
    const int lane = threadIdx.x & 31;
    const long long r = (long long)blockIdx.x * CLS_WARPS + (threadIdx.x >> 5);
    if (r >= R) return;
    const bf16* xr = x + r * ldx;
    const unsigned long long g0 = (unsigned long long)r * (unsigned)(H >> 5);     // group32 of element r*H + col: g0 + col / 32
    for (int l0 = 0; l0 < L; l0 += CLS_LC) {
        float acc[CLS_LC] = {0.f, 0.f, 0.f, 0.f};
        for (int col = lane * 8; col < H; col += 256) {
            float xv[8];
            unpack8(ld_global_nc_v4(xr + col), xv);
            if (thresh != 0u) {
                const uint32_t keep = dropout_keep8(seed, stream_id, g0 + (col >> 5), (col & 31) >> 3, thresh);
#pragma unroll
                for (int i = 0; i < 8; ++i) xv[i] = ((keep >> i) & 1u) ? xv[i] * drop_scale : 0.f;
            }
#pragma unroll
            for (int j = 0; j < CLS_LC; ++j) {
                if (l0 + j < L) {
                    float wv[8];
                    unpack8(ld_global_nc_v4(w + (long long)(l0 + j) * H + col), wv);
#pragma unroll
                    for (int i = 0; i < 8; ++i) acc[j] = fmaf(xv[i], wv[i], acc[j]);
                }
            }
        }
#pragma unroll
        for (int j = 0; j < CLS_LC; ++j) {
            const float s = warp_sum(acc[j]);
            if (lane == j && l0 + j < L) st_f32(logits + r * L + l0 + j, s + ld_f32(b + l0 + j));
        }
    }
}

// backward: CTA (column block of CLSB_THREADS, slab of CLSB_ROWS rows), one thread per column.  dx is written per element; dW and db
// go to per-slab fp32 partials (rows in order), which colsum_finalize_kernel sums over slabs in a fixed order: no atomics.
constexpr int CLSB_THREADS = 256, CLSB_ROWS = 32;
template <typename T, int LMAX>
__global__ void __launch_bounds__(CLSB_THREADS)
cls_head_bwd_kernel(const T* __restrict__ dlogits, const bf16* __restrict__ x, long long ldx, const bf16* __restrict__ w, int R, int H,
                    int L, uint32_t thresh, float drop_scale, unsigned long long seed, const unsigned long long* seed_dev,
                    uint32_t stream_id, bf16* __restrict__ dx, float* __restrict__ part_dw, float* __restrict__ part_db) {
    __shared__ float d_s[CLSB_ROWS][LMAX];
    seed = effective_seed(seed, seed_dev);
    const long long r0 = (long long)blockIdx.y * CLSB_ROWS;
    const int nr = (int)min((long long)CLSB_ROWS, R - r0);
    for (int i = threadIdx.x; i < CLSB_ROWS * LMAX; i += CLSB_THREADS) {
        const int rr = i / LMAX, l = i % LMAX;
        d_s[rr][l] = (rr < nr && l < L) ? ld_f32(dlogits + (r0 + rr) * L + l) : 0.f;
    }
    __syncthreads();
    if (blockIdx.x == 0 && threadIdx.x < L) {
        float s = 0.f;
        for (int rr = 0; rr < nr; ++rr) s += d_s[rr][threadIdx.x];
        part_db[(long long)blockIdx.y * L + threadIdx.x] = s;
    }
    const int c = blockIdx.x * CLSB_THREADS + threadIdx.x;
    if (c >= H) return;
    float wc[LMAX], acc[LMAX];
#pragma unroll
    for (int l = 0; l < LMAX; ++l) {
        wc[l] = l < L ? __bfloat162float(w[(long long)l * H + c]) : 0.f;
        acc[l] = 0.f;
    }
    for (int rr = 0; rr < nr; ++rr) {
        const long long r = r0 + rr;
        const float xv = __bfloat162float(x[r * ldx + c]);
        bool kept = true;
        float sc = 1.f;
        if (thresh != 0u) {
            kept = (dropout_keep8(seed, stream_id, (unsigned long long)(r * H + c) >> 5, (c & 31) >> 3, thresh) >> (c & 7)) & 1u;
            sc = drop_scale;
        }
        const float xd = kept ? xv * sc : 0.f;
        float g = 0.f;
#pragma unroll
        for (int l = 0; l < LMAX; ++l) {
            if (l < L) {
                const float d = d_s[rr][l];
                g = fmaf(d, wc[l], g);
                acc[l] = fmaf(d, xd, acc[l]);
            }
        }
        dx[r * H + c] = __float2bfloat16_rn(kept ? g * sc : 0.f);
    }
#pragma unroll
    for (int l = 0; l < LMAX; ++l)
        if (l < L) part_dw[((long long)blockIdx.y * L + l) * H + c] = acc[l];
}
__global__ void cast_f32_bf16_kernel(const float* __restrict__ x, bf16* __restrict__ y, long long n) {
    const long long nv = n / 4;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nv; i += (long long)gridDim.x * blockDim.x) {
        float4 f = *reinterpret_cast<const float4*>(x + i * 4);
        *reinterpret_cast<uint2*>(y + i * 4) = make_uint2(pack_bf16(f.x, f.y), pack_bf16(f.z, f.w));
    }
    if (blockIdx.x == 0 && threadIdx.x < (n & 3)) y[nv * 4 + threadIdx.x] = __float2bfloat16_rn(x[nv * 4 + threadIdx.x]);
}
__global__ void cast_bf16_f32_kernel(const bf16* __restrict__ x, float* __restrict__ y, long long n) {
    const long long nv = n / 4;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nv; i += (long long)gridDim.x * blockDim.x) {
        uint2 u = *reinterpret_cast<const uint2*>(x + i * 4);
        float2 a = unpack_bf16(u.x), b = unpack_bf16(u.y);
        *reinterpret_cast<float4*>(y + i * 4) = make_float4(a.x, a.y, b.x, b.y);
    }
    if (blockIdx.x == 0 && threadIdx.x < (n & 3)) y[nv * 4 + threadIdx.x] = __bfloat162float(x[nv * 4 + threadIdx.x]);
}

static int ew_grid(long long work_items, int threads) {
    long long g = (work_items + threads - 1) / threads, cap = (long long)sm_count() * 8;
    return (int)(g < cap ? (g > 0 ? g : 1) : cap);
}

}  // namespace dle

using namespace dle;
#define S_(x) reinterpret_cast<cudaStream_t>(x)
#define B_(x) reinterpret_cast<const bf16*>(x)
#define BM_(x) reinterpret_cast<bf16*>(x)
#define ALIGNED16(p) ((reinterpret_cast<uintptr_t>(p) & 15) == 0)

#define LN_DISPATCH(H, CALL)                                  \
    switch ((H) / 256) {                                      \
        case 1: { constexpr int J = 1; CALL; break; }         \
        case 2: { constexpr int J = 2; CALL; break; }         \
        case 3: { constexpr int J = 3; CALL; break; }         \
        case 4: { constexpr int J = 4; CALL; break; }         \
        default: return DLE_ERR_INVALID;                      \
    }

extern "C" int dle_add_ln_fwd(const void* x, const void* bias, const void* residual, const void* gamma, const void* beta,
                              void* z_out, void* y, float* mean, float* rstd, int64_t T, int32_t H, float eps,
                              float dropout_p, uint64_t seed, const uint64_t* seed_dev, uint32_t dropout_stream, void* stream) {
    DLE_CHECK_ARG(x && gamma && beta && y && mean && rstd && T > 0 && H > 0 && H % 256 == 0 && H <= 1024);
    DLE_CHECK_ARG(ALIGNED16(x) && ALIGNED16(y) && ALIGNED16(gamma) && ALIGNED16(beta) && ALIGNED16(bias) && ALIGNED16(residual) && ALIGNED16(z_out));
    DLE_CHECK_ARG(dropout_p >= 0.f && dropout_p < 1.f);
    if (bias || residual || dropout_p > 0.f) DLE_CHECK_ARG(z_out != nullptr);
    const uint32_t th = dropout_p > 0.f ? dropout_thresh16(dropout_p) : 0u;
    const float sc = dropout_p > 0.f ? 1.f / (1.f - dropout_p) : 1.f;
    if (H % 512 == 0 && !ln_force_one_warp()) {
        if (H == 1024) add_ln_fwd2_kernel<2><<<ln2_grid(T), LN2_THREADS, 0, S_(stream)>>>(B_(x), B_(bias), B_(residual), B_(gamma), B_(beta), BM_(z_out), BM_(y), mean, rstd, T, eps, th, sc, seed, reinterpret_cast<const unsigned long long*>(seed_dev), dropout_stream);
        else add_ln_fwd2_kernel<1><<<ln2_grid(T), LN2_THREADS, 0, S_(stream)>>>(B_(x), B_(bias), B_(residual), B_(gamma), B_(beta), BM_(z_out), BM_(y), mean, rstd, T, eps, th, sc, seed, reinterpret_cast<const unsigned long long*>(seed_dev), dropout_stream);
        DLE_LAUNCH_CHECK();
        return DLE_OK;
    }
    LN_DISPATCH(H, (add_ln_fwd_kernel<J><<<ln_grid(T), LN_THREADS, 0, S_(stream)>>>(B_(x), B_(bias), B_(residual), B_(gamma), B_(beta),
                    BM_(z_out), BM_(y), mean, rstd, T, eps, th, sc, seed, reinterpret_cast<const unsigned long long*>(seed_dev), dropout_stream)));
    DLE_LAUNCH_CHECK();
    return DLE_OK;
}

// upper bound valid for both kernel families (the caller sizes the partial workspace with it; rows beyond the launched grid
// are simply not written and dle_colsum_finalize is given the actual count through dle_ln_bwd_partials_h)
extern "C" int dle_ln_bwd_partials(int64_t T) { int a = ln_grid(T), b = ln2_grid(T); return a > b ? a : b; }
extern "C" int dle_ln_bwd_partials_h(int64_t T, int32_t H) { return (H % 512 == 0 && !ln_force_one_warp()) ? ln2_grid(T) : ln_grid(T); }

extern "C" int dle_add_ln_bwd(const void* dy, const void* z, const float* mean, const float* rstd, const void* gamma,
                              void* dz_out, void* dx_out, float* part_dgamma, float* part_dbeta, float* part_dbias,
                              int64_t T, int32_t H, float dropout_p, uint64_t seed, const uint64_t* seed_dev, uint32_t dropout_stream, void* stream) {
    DLE_CHECK_ARG(dy && z && mean && rstd && gamma && T > 0 && H > 0 && H % 256 == 0 && H <= 1024);
    DLE_CHECK_ARG(ALIGNED16(dy) && ALIGNED16(z) && ALIGNED16(gamma) && ALIGNED16(dz_out) && ALIGNED16(dx_out));
    DLE_CHECK_ARG(dz_out != nullptr || dx_out != nullptr);
    DLE_CHECK_ARG(dropout_p >= 0.f && dropout_p < 1.f);
    if (dropout_p > 0.f) DLE_CHECK_ARG(dx_out != nullptr);
    if (dropout_p == 0.f && dz_out == nullptr) { dz_out = dx_out; dx_out = nullptr; }   // dx == dz without dropout
    const uint32_t th = dropout_p > 0.f ? dropout_thresh16(dropout_p) : 0u;
    const float sc = dropout_p > 0.f ? 1.f / (1.f - dropout_p) : 1.f;
    if (H % 512 == 0 && !ln_force_one_warp()) {
        if (int rc = (H == 1024 ? ln2_bwd_attr<2>() : ln2_bwd_attr<1>())) return rc;
        if (H == 1024) add_ln_bwd2_kernel<2><<<ln2_grid(T), LN2_THREADS, ln2_bwd_smem(2), S_(stream)>>>(B_(dy), B_(z), mean, rstd, B_(gamma), BM_(dz_out), BM_(dx_out), part_dgamma, part_dbeta, part_dbias, T, th, sc, seed, reinterpret_cast<const unsigned long long*>(seed_dev), dropout_stream);
        else add_ln_bwd2_kernel<1><<<ln2_grid(T), LN2_THREADS, ln2_bwd_smem(1), S_(stream)>>>(B_(dy), B_(z), mean, rstd, B_(gamma), BM_(dz_out), BM_(dx_out), part_dgamma, part_dbeta, part_dbias, T, th, sc, seed, reinterpret_cast<const unsigned long long*>(seed_dev), dropout_stream);
        DLE_LAUNCH_CHECK();
        return DLE_OK;
    }
    LN_DISPATCH(H, (add_ln_bwd_kernel<J><<<ln_grid(T), LN_THREADS, 0, S_(stream)>>>(B_(dy), B_(z), mean, rstd, B_(gamma), BM_(dz_out),
                    BM_(dx_out), part_dgamma, part_dbeta, part_dbias, T, th, sc, seed, reinterpret_cast<const unsigned long long*>(seed_dev), dropout_stream)));
    DLE_LAUNCH_CHECK();
    return DLE_OK;
}

extern "C" int dle_colsum_finalize(const float* part, int32_t n_part, int32_t N, void* out, int32_t out_dtype,
                                   int32_t accumulate, void* stream) {
    return dle_colsum_finalize_batched(part, 1, n_part, N, out, out_dtype, accumulate, stream);
}
extern "C" int dle_colsum_finalize_batched(const float* part, int32_t n_arrays, int32_t n_part, int32_t N, void* out,
                                           int32_t out_dtype, int32_t accumulate, void* stream) {
    DLE_CHECK_ARG(part && out && n_arrays > 0 && n_part > 0 && N > 0 && (out_dtype == DLE_DTYPE_F32 || out_dtype == DLE_DTYPE_BF16));
    colsum_finalize_kernel<<<dim3((N + 31) / 32, n_arrays), CF_WARPS * 32, 0, S_(stream)>>>(part, n_part, N, out, out_dtype, accumulate);
    DLE_LAUNCH_CHECK();
    return DLE_OK;
}

static int colsum_rows_per_slab(int64_t T) { long long r = (T + 127) / 128; return (int)(r < 32 ? 32 : r); }
extern "C" int dle_colsum_partials(int64_t T) { int r = colsum_rows_per_slab(T); return (int)((T + r - 1) / r); }
extern "C" int dle_colsum_bf16(const void* x, int64_t T, int32_t N, int64_t ldx, float* part, void* stream) {
    DLE_CHECK_ARG(x && part && T > 0 && N > 0 && N % 8 == 0 && ldx % 8 == 0 && ALIGNED16(x));
    const int r = colsum_rows_per_slab(T);
    dim3 grid((N + 255) / 256, (unsigned)((T + r - 1) / r));
    colsum_bf16_kernel<<<grid, CS_WARPS * 32, 0, S_(stream)>>>(B_(x), T, N, ldx, part, r);
    DLE_LAUNCH_CHECK();
    return DLE_OK;
}

extern "C" int dle_bias_gelu_fwd(const void* x, const void* bias, void* u_out, void* y, int64_t T, int32_t N, void* stream) {
    DLE_CHECK_ARG(x && y && T > 0 && N > 0 && N % 8 == 0 && ALIGNED16(x) && ALIGNED16(y) && ALIGNED16(bias) && ALIGNED16(u_out));
    bias_gelu_fwd_kernel<<<ew_grid(T * N / 8, 256), 256, 0, S_(stream)>>>(B_(x), B_(bias), BM_(u_out), BM_(y), T, N);
    DLE_LAUNCH_CHECK();
    return DLE_OK;
}
extern "C" int dle_bias_gelu_bwd(const void* dy, const void* u, void* du, int64_t T, int32_t N, void* stream) {
    DLE_CHECK_ARG(dy && u && du && T > 0 && N > 0 && (T * N) % 8 == 0 && ALIGNED16(dy) && ALIGNED16(u) && ALIGNED16(du));
    bias_gelu_bwd_kernel<<<ew_grid(T * N / 8, 256), 256, 0, S_(stream)>>>(B_(dy), B_(u), BM_(du), T * N / 8);
    DLE_LAUNCH_CHECK();
    return DLE_OK;
}

extern "C" int dle_embed_ln_fwd(const int64_t* input_ids, const int64_t* token_type_ids, const void* word, const void* pos,
                                const void* type, const void* gamma, const void* beta, void* z_out, void* y, float* mean,
                                float* rstd, int32_t B, int32_t S, int32_t H, int32_t V, int32_t P, int32_t NT, float eps,
                                float dropout_p, uint64_t seed, const uint64_t* seed_dev, uint32_t dropout_stream, int32_t* err_flag, void* stream,
                                const int64_t* position_ids) {
    DLE_CHECK_ARG(input_ids && token_type_ids && word && pos && type && gamma && beta && y && mean && rstd);
    DLE_CHECK_ARG(B > 0 && S > 0 && H % 256 == 0 && H > 0 && H <= 1024 && V > 0 && P >= S && NT > 0);
    DLE_CHECK_ARG(ALIGNED16(word) && ALIGNED16(pos) && ALIGNED16(type) && ALIGNED16(y) && ALIGNED16(z_out) && ALIGNED16(gamma) && ALIGNED16(beta));
    DLE_CHECK_ARG(dropout_p >= 0.f && dropout_p < 1.f && (reinterpret_cast<uintptr_t>(position_ids) & 7) == 0);
    const uint32_t th = dropout_p > 0.f ? dropout_thresh16(dropout_p) : 0u;
    const float sc = dropout_p > 0.f ? 1.f / (1.f - dropout_p) : 1.f;
    const long long T = (long long)B * S;
    LN_DISPATCH(H, (embed_ln_fwd_kernel<J><<<ln_grid(T), LN_THREADS, 0, S_(stream)>>>(
                    reinterpret_cast<const long long*>(input_ids), reinterpret_cast<const long long*>(token_type_ids), B_(word), B_(pos),
                    B_(type), B_(gamma), B_(beta), BM_(z_out), BM_(y), mean, rstd, B, S, V, P, NT, eps, th, sc, seed, reinterpret_cast<const unsigned long long*>(seed_dev), dropout_stream, err_flag,
                    reinterpret_cast<const long long*>(position_ids))));
    DLE_LAUNCH_CHECK();
    return DLE_OK;
}

extern "C" int dle_embed_ln_bwd(const void* dy, const void* z, const float* mean, const float* rstd, const void* gamma,
                                const int64_t* input_ids, const int64_t* token_type_ids, float* dword, float* dpos,
                                float* dtype_tab, float* part_dgamma, float* part_dbeta, int32_t B, int32_t S, int32_t H,
                                float dropout_p, uint64_t seed, const uint64_t* seed_dev, uint32_t dropout_stream, void* stream,
                                const int64_t* position_ids) {
    DLE_CHECK_ARG(dy && z && mean && rstd && gamma && input_ids && token_type_ids && dword && dpos && dtype_tab && part_dgamma && part_dbeta);
    DLE_CHECK_ARG(B > 0 && S > 0 && H % 256 == 0 && H > 0 && H <= 1024 && ALIGNED16(dy) && ALIGNED16(z) && ALIGNED16(dword) && ALIGNED16(dpos) && ALIGNED16(dtype_tab));
    DLE_CHECK_ARG((reinterpret_cast<uintptr_t>(position_ids) & 7) == 0);
    const uint32_t th = dropout_p > 0.f ? dropout_thresh16(dropout_p) : 0u;
    const float sc = dropout_p > 0.f ? 1.f / (1.f - dropout_p) : 1.f;
    const long long T = (long long)B * S;
    LN_DISPATCH(H, (embed_ln_bwd_kernel<J><<<ln_grid(T), LN_THREADS, 0, S_(stream)>>>(
                    B_(dy), B_(z), mean, rstd, B_(gamma), reinterpret_cast<const long long*>(input_ids),
                    reinterpret_cast<const long long*>(token_type_ids), dword, dpos, dtype_tab, part_dgamma, part_dbeta, B, S, th, sc,
                    seed, reinterpret_cast<const unsigned long long*>(seed_dev), dropout_stream, reinterpret_cast<const long long*>(position_ids))));
    DLE_LAUNCH_CHECK();
    return DLE_OK;
}

extern "C" int dle_gather_rows(const void* x, const int64_t* idx, void* out, int64_t n_idx, int32_t H, int64_t n_rows,
                               int32_t* err_flag, void* stream) {
    DLE_CHECK_ARG(x && idx && out && n_idx >= 0 && H > 0 && H % 8 == 0 && n_rows > 0 && ALIGNED16(x) && ALIGNED16(out));
    if (n_idx == 0) return DLE_OK;
    gather_rows_kernel<<<ew_grid(n_idx * (H / 8), 256), 256, 0, S_(stream)>>>(B_(x), reinterpret_cast<const long long*>(idx), BM_(out), n_idx, H, n_rows, err_flag);
    DLE_LAUNCH_CHECK();
    return DLE_OK;
}
extern "C" int dle_scatter_rows(const void* dy, const int64_t* idx, void* dx, int64_t n_idx, int32_t H, int64_t n_rows, void* stream) {
    DLE_CHECK_ARG(dy && idx && dx && n_idx >= 0 && H > 0 && H % 8 == 0 && n_rows > 0 && ALIGNED16(dy) && ALIGNED16(dx));
    if (n_idx == 0) return DLE_OK;
    scatter_rows_kernel<<<ew_grid(n_idx * (H / 8), 256), 256, 0, S_(stream)>>>(B_(dy), reinterpret_cast<const long long*>(idx), BM_(dx), n_idx, H, n_rows);
    DLE_LAUNCH_CHECK();
    return DLE_OK;
}
extern "C" int dle_segment_table(const int64_t* mask, int32_t B, int32_t S, int32_t k, int32_t* cu_seqlens, int64_t* position_ids,
                                 int64_t* cls_index, int32_t* err_flag, void* stream) {
    DLE_CHECK_ARG(mask && cu_seqlens && position_ids && cls_index && B > 0 && S > 0 && k > 0);
    DLE_CHECK_ARG((long long)B * (k + 1) <= 65535 && (long long)B * S <= 0x7fffffffLL);
    DLE_CHECK_ARG(((reinterpret_cast<uintptr_t>(mask) | reinterpret_cast<uintptr_t>(position_ids) | reinterpret_cast<uintptr_t>(cls_index)) & 7) == 0);
    DLE_CHECK_ARG((reinterpret_cast<uintptr_t>(cu_seqlens) & 3) == 0 && (reinterpret_cast<uintptr_t>(err_flag) & 3) == 0);
    segment_table_kernel<<<(B + SEG_WARPS - 1) / SEG_WARPS, SEG_WARPS * 32, 0, S_(stream)>>>(
        reinterpret_cast<const long long*>(mask), B, S, k, cu_seqlens, reinterpret_cast<long long*>(position_ids),
        reinterpret_cast<long long*>(cls_index), err_flag);
    DLE_LAUNCH_CHECK();
    return DLE_OK;
}
static bool span_logits_args_ok(const void* a, const void* b, const void* c, const int32_t* cu_seqlens, int32_t B, int32_t S, int32_t k,
                                int32_t dtype, int64_t ld) {
    if (!(a && b && c && cu_seqlens && B > 0 && S > 0 && k > 0 && ld >= 2)) return false;
    if ((long long)B * (k + 1) > 65535 || (long long)B * S > 0x7fffffffLL) return false;
    if (dtype != DLE_DTYPE_F32 && dtype != DLE_DTYPE_BF16) return false;
    const uintptr_t align = dtype == DLE_DTYPE_F32 ? 3 : 1;
    return ((reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(b) | reinterpret_cast<uintptr_t>(c)) & align) == 0 &&
           (reinterpret_cast<uintptr_t>(cu_seqlens) & 3) == 0;
}
extern "C" int dle_span_logits_unpack(const void* logits, int64_t ld, const int32_t* cu_seqlens, int32_t B, int32_t S, int32_t k,
                                      int32_t dtype, float fill, void* start_out, void* end_out, void* stream) {
    DLE_CHECK_ARG(span_logits_args_ok(logits, start_out, end_out, cu_seqlens, B, S, k, dtype, ld));
    const long long n = (long long)B * k * S;
    if (dtype == DLE_DTYPE_F32)
        span_logits_unpack_kernel<float><<<ew_grid(n, 256), 256, 0, S_(stream)>>>(
            reinterpret_cast<const float*>(logits), ld, cu_seqlens, S, k, n, fill, reinterpret_cast<float*>(start_out),
            reinterpret_cast<float*>(end_out));
    else
        span_logits_unpack_kernel<bf16><<<ew_grid(n, 256), 256, 0, S_(stream)>>>(B_(logits), ld, cu_seqlens, S, k, n, fill,
                                                                                  BM_(start_out), BM_(end_out));
    DLE_LAUNCH_CHECK();
    return DLE_OK;
}
extern "C" int dle_span_logits_pack_grad(const void* dstart, const void* dend, const int32_t* cu_seqlens, int32_t B, int32_t S, int32_t k,
                                         int32_t dtype, void* dlogits, int64_t ld, void* stream) {
    DLE_CHECK_ARG(span_logits_args_ok(dstart, dend, dlogits, cu_seqlens, B, S, k, dtype, ld));
    const long long n = (long long)B * S;
    if (dtype == DLE_DTYPE_F32)
        span_logits_pack_grad_kernel<float><<<ew_grid(n, 256), 256, 0, S_(stream)>>>(
            reinterpret_cast<const float*>(dstart), reinterpret_cast<const float*>(dend), cu_seqlens, S, k, n,
            reinterpret_cast<float*>(dlogits), ld);
    else
        span_logits_pack_grad_kernel<bf16><<<ew_grid(n, 256), 256, 0, S_(stream)>>>(B_(dstart), B_(dend), cu_seqlens, S, k, n,
                                                                                     BM_(dlogits), ld);
    DLE_LAUNCH_CHECK();
    return DLE_OK;
}
static bool cls_head_args_ok(const void* x, int64_t ldx, const void* w, int32_t R, int32_t H, int32_t L, int32_t dtype, float dropout_p) {
    if (!(x && w && R > 0 && H > 0 && H % 32 == 0 && L >= 1 && L <= 32 && ldx >= H && ldx % 8 == 0)) return false;
    if ((long long)R > 65535LL * CLSB_ROWS || (dtype != DLE_DTYPE_F32 && dtype != DLE_DTYPE_BF16)) return false;
    return dropout_p >= 0.f && dropout_p < 1.f && ALIGNED16(x) && ALIGNED16(w);
}
static bool dtype_aligned(const void* p, int32_t dtype) {
    return (reinterpret_cast<uintptr_t>(p) & (dtype == DLE_DTYPE_F32 ? 3 : 1)) == 0;
}
extern "C" int dle_cls_head_fwd(const void* x, int64_t ldx, const void* w, const void* b, int32_t R, int32_t H, int32_t L, int32_t dtype,
                                float dropout_p, uint64_t seed, const uint64_t* seed_dev, uint32_t dropout_stream, void* logits,
                                void* stream) {
    DLE_CHECK_ARG(cls_head_args_ok(x, ldx, w, R, H, L, dtype, dropout_p) && b && logits);
    DLE_CHECK_ARG(dtype_aligned(b, dtype) && dtype_aligned(logits, dtype));
    const uint32_t th = dropout_p > 0.f ? dropout_thresh16(dropout_p) : 0u;
    const float sc = dropout_p > 0.f ? 1.f / (1.f - dropout_p) : 1.f;
    const auto sdev = reinterpret_cast<const unsigned long long*>(seed_dev);
    const int grid = (R + CLS_WARPS - 1) / CLS_WARPS;
    if (dtype == DLE_DTYPE_F32)
        cls_head_fwd_kernel<float><<<grid, CLS_WARPS * 32, 0, S_(stream)>>>(B_(x), ldx, B_(w), reinterpret_cast<const float*>(b), R, H, L,
                                                                            th, sc, seed, sdev, dropout_stream, reinterpret_cast<float*>(logits));
    else
        cls_head_fwd_kernel<bf16><<<grid, CLS_WARPS * 32, 0, S_(stream)>>>(B_(x), ldx, B_(w), B_(b), R, H, L, th, sc, seed, sdev,
                                                                           dropout_stream, BM_(logits));
    DLE_LAUNCH_CHECK();
    return DLE_OK;
}
extern "C" int dle_cls_head_bwd_partials(int32_t R) { return R > 0 ? (R + CLSB_ROWS - 1) / CLSB_ROWS : DLE_ERR_INVALID; }
extern "C" int dle_cls_head_bwd(const void* dlogits, const void* x, int64_t ldx, const void* w, int32_t R, int32_t H, int32_t L,
                                int32_t dtype, float dropout_p, uint64_t seed, const uint64_t* seed_dev, uint32_t dropout_stream, void* dx,
                                float* part, void* dw, void* db, void* stream) {
    DLE_CHECK_ARG(cls_head_args_ok(x, ldx, w, R, H, L, dtype, dropout_p) && dlogits && dx && part && dw && db);
    DLE_CHECK_ARG(dtype_aligned(dlogits, dtype) && dtype_aligned(dw, dtype) && dtype_aligned(db, dtype));
    DLE_CHECK_ARG((reinterpret_cast<uintptr_t>(dx) & 1) == 0 && (reinterpret_cast<uintptr_t>(part) & 3) == 0);
    const uint32_t th = dropout_p > 0.f ? dropout_thresh16(dropout_p) : 0u;
    const float sc = dropout_p > 0.f ? 1.f / (1.f - dropout_p) : 1.f;
    const auto sdev = reinterpret_cast<const unsigned long long*>(seed_dev);
    const int n_part = (R + CLSB_ROWS - 1) / CLSB_ROWS;
    float* part_dw = part;
    float* part_db = part + (long long)n_part * L * H;
    const dim3 grid((H + CLSB_THREADS - 1) / CLSB_THREADS, n_part);
#define CLS_BWD(T, LM, D) cls_head_bwd_kernel<T, LM><<<grid, CLSB_THREADS, 0, S_(stream)>>>(D, B_(x), ldx, B_(w), R, H, L, th, sc, seed, \
                                                                                         sdev, dropout_stream, BM_(dx), part_dw, part_db)
    const float* d32 = reinterpret_cast<const float*>(dlogits);
    if (dtype == DLE_DTYPE_F32) { if (L <= 4) CLS_BWD(float, 4, d32); else CLS_BWD(float, 32, d32); }
    else { if (L <= 4) CLS_BWD(bf16, 4, B_(dlogits)); else CLS_BWD(bf16, 32, B_(dlogits)); }
#undef CLS_BWD
    DLE_LAUNCH_CHECK();
    if (int rc = dle_colsum_finalize(part_dw, n_part, L * H, dw, dtype, 0, stream)) return rc;
    return dle_colsum_finalize(part_db, n_part, L, db, dtype, 0, stream);
}
__global__ void advance_u64_kernel(unsigned long long* c, unsigned long long d) { *c += d; }
extern "C" int dle_advance_u64(uint64_t* counter, uint64_t delta, void* stream) {
    DLE_CHECK_ARG(counter && (reinterpret_cast<uintptr_t>(counter) & 7) == 0);
    advance_u64_kernel<<<1, 1, 0, S_(stream)>>>(reinterpret_cast<unsigned long long*>(counter), delta);
    DLE_LAUNCH_CHECK();
    return DLE_OK;
}
extern "C" int dle_cast_f32_to_bf16(const float* x, void* y, int64_t n, void* stream) {
    DLE_CHECK_ARG(x && y && n > 0 && ALIGNED16(x) && (reinterpret_cast<uintptr_t>(y) & 7) == 0);
    cast_f32_bf16_kernel<<<ew_grid(n / 4 + 1, 256), 256, 0, S_(stream)>>>(x, BM_(y), n);
    DLE_LAUNCH_CHECK();
    return DLE_OK;
}
extern "C" int dle_cast_bf16_to_f32(const void* x, float* y, int64_t n, void* stream) {
    DLE_CHECK_ARG(x && y && n > 0 && ALIGNED16(y) && (reinterpret_cast<uintptr_t>(x) & 7) == 0);
    cast_bf16_f32_kernel<<<ew_grid(n / 4 + 1, 256), 256, 0, S_(stream)>>>(B_(x), y, n);
    DLE_LAUNCH_CHECK();
    return DLE_OK;
}

extern "C" int dle_version(char* host_buf, int host_buf_len) {
    static const char v[] = "dle_b200 0.2 sm_90a";
    if (host_buf && host_buf_len > 0) {
        int i = 0;
        for (; i < host_buf_len - 1 && v[i]; ++i) host_buf[i] = v[i];
        host_buf[i] = 0;
    }
    return 90;
}
