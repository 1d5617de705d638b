// Softmax cross-entropy over the vocabulary on bf16 logits with fp32 arithmetic, forward and backward, one CTA per row.
//
// replaces the criterion's CrossEntropyLoss(ignore_index=-1) on the MLM logits
// (PyTorch/LanguageModeling/BERT/run_pretraining.py:85-95): under the reference's autocast that op up-casts the [rows, V] fp16
// logits to fp32, runs log_softmax + nll_loss forward and their backward -- four passes over a 1.25 GB fp32 tensor at rows = 10240,
// V = 30528.  Here the bf16 row (61 KB) is read once per direction and all arithmetic happens in fp32 registers:
//   fwd: lse[r] = log sum_v exp(x[r,v]) ; loss[r] = lse[r] - x[r, label[r]]   (0 for ignored rows)
//   bwd: dx[r,v] = (exp(x[r,v] - lse[r]) - [v == label[r]]) * g            (g = dLoss / number of counted rows, a DEVICE scalar)
// HBM-bound: 2*rows*V bytes forward, 4*rows*V backward.
#include "common.cuh"
#include "../../include/dle_b200.h"

namespace dle {

constexpr int CE_THREADS = 256;
constexpr int CE_MAX_VEC = 16;                  // 16-byte vectors per thread held in registers: V <= 256 * 16 * 8 = 32768

__device__ __forceinline__ float block_max(float v, float* sh) {
    v = warp_max(v);
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
    __syncthreads();
    if (l == 0) sh[w] = v;
    __syncthreads();
    float r = sh[0];
#pragma unroll
    for (int i = 1; i < CE_THREADS / 32; ++i) r = fmaxf(r, sh[i]);
    return r;
}
__device__ __forceinline__ float block_sum(float v, float* sh) {
    v = warp_sum(v);
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
    __syncthreads();
    if (l == 0) sh[w] = v;
    __syncthreads();
    float r = 0.f;
#pragma unroll
    for (int i = 0; i < CE_THREADS / 32; ++i) r += sh[i];
    return r;
}
__device__ __forceinline__ void unpack8f(const uint4& u, float* f) {
    float2 a = unpack_bf16(u.x), b = unpack_bf16(u.y), c = unpack_bf16(u.z), d = unpack_bf16(u.w);
    f[0] = a.x; f[1] = a.y; f[2] = b.x; f[3] = b.y; f[4] = c.x; f[5] = c.y; f[6] = d.x; f[7] = d.y;
}

__global__ void __launch_bounds__(CE_THREADS)
softmax_ce_fwd_kernel(const bf16* __restrict__ x, const long long* __restrict__ labels, float* __restrict__ lse_out,
                      float* __restrict__ loss_out, long long rows, int V, long long ldx, long long ignore_index, int* err_flag) {
    __shared__ float sh[CE_THREADS / 32];
    const int nvec = V / 8;
    for (long long r = blockIdx.x; r < rows; r += gridDim.x) {
        const bf16* row = x + r * ldx;
        uint4 buf[CE_MAX_VEC];
        float mx = -INFINITY;
#pragma unroll
        for (int i = 0; i < CE_MAX_VEC; ++i) {
            const int v = threadIdx.x + i * CE_THREADS;
            if (v < nvec) {
                buf[i] = ld_global_nc_v4(row + v * 8);
                float f[8];
                unpack8f(buf[i], f);
#pragma unroll
                for (int k = 0; k < 8; ++k) mx = fmaxf(mx, f[k]);
            }
        }
        mx = block_max(mx, sh);
        float s = 0.f;
        const float mxl = mx * 1.4426950408889634f;
#pragma unroll
        for (int i = 0; i < CE_MAX_VEC; ++i) {
            const int v = threadIdx.x + i * CE_THREADS;
            if (v < nvec) {
                float f[8];
                unpack8f(buf[i], f);
#pragma unroll
                for (int k = 0; k < 8; ++k) s += exp2f(fmaf(f[k], 1.4426950408889634f, -mxl));
            }
        }
        s = block_sum(s, sh);
        if (threadIdx.x == 0) {
            const float lse = mx + logf(s);
            lse_out[r] = lse;
            const long long lab = labels[r];
            float loss = 0.f;
            if (lab != ignore_index) {
                if (lab < 0 || lab >= V) { if (err_flag) atomicExch(err_flag, 1); }
                else loss = lse - __bfloat162float(row[lab]);
            }
            loss_out[r] = loss;
        }
    }
}

__global__ void __launch_bounds__(CE_THREADS)
softmax_ce_bwd_kernel(const bf16* __restrict__ x, const long long* __restrict__ labels, const float* __restrict__ lse,
                      const float* __restrict__ gscale, bf16* __restrict__ dx, long long rows, int V, long long ldx, long long lddx,
                      long long ignore_index) {
    const int nvec = V / 8;
    const float g = *gscale;
    for (long long r = blockIdx.x; r < rows; r += gridDim.x) {
        const bf16* row = x + r * ldx;
        bf16* drow = dx + r * lddx;
        const long long lab = labels[r];
        const bool counted = lab != ignore_index && lab >= 0 && lab < V;
        const float nl = -lse[r] * 1.4426950408889634f;
        for (int v = threadIdx.x; v < nvec; v += CE_THREADS) {
            float f[8];
            if (counted) {
                unpack8f(ld_global_nc_v4(row + v * 8), f);
#pragma unroll
                for (int k = 0; k < 8; ++k) {
                    float p = exp2f(fmaf(f[k], 1.4426950408889634f, nl));
                    if ((long long)(v * 8 + k) == lab) p -= 1.0f;
                    f[k] = p * g;
                }
            } else {
#pragma unroll
                for (int k = 0; k < 8; ++k) f[k] = 0.f;
            }
            st_global_v4(drow + v * 8, pack_bf16(f[0], f[1]), pack_bf16(f[2], f[3]), pack_bf16(f[4], f[5]), pack_bf16(f[6], f[7]));
        }
    }
}

}  // namespace dle

using namespace dle;

static int ce_grid(long long rows) {
    int dev = 0, sms = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    const long long cap = (long long)sms * 8;
    return (int)(rows < cap ? rows : cap);
}

extern "C" int dle_softmax_ce_fwd(const void* logits, const int64_t* labels, float* lse, float* loss_rows, int64_t rows, int32_t V,
                                  int64_t ld, int64_t ignore_index, int32_t* err_flag, void* stream) {
    DLE_CHECK_ARG(logits && labels && lse && loss_rows && rows >= 0 && V > 0 && V % 8 == 0 && V <= CE_THREADS * CE_MAX_VEC * 8);
    DLE_CHECK_ARG(ld >= V && ld % 8 == 0 && (reinterpret_cast<uintptr_t>(logits) & 15) == 0);
    if (rows == 0) return DLE_OK;
    softmax_ce_fwd_kernel<<<ce_grid(rows), CE_THREADS, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
        reinterpret_cast<const bf16*>(logits), reinterpret_cast<const long long*>(labels), lse, loss_rows, rows, V, ld, ignore_index, err_flag);
    DLE_LAUNCH_CHECK();
    return DLE_OK;
}

extern "C" int dle_softmax_ce_bwd(const void* logits, const int64_t* labels, const float* lse, const float* grad_scale, void* dlogits,
                                  int64_t rows, int32_t V, int64_t ld, int64_t ld_d, int64_t ignore_index, void* stream) {
    DLE_CHECK_ARG(logits && labels && lse && grad_scale && dlogits && rows >= 0 && V > 0 && V % 8 == 0);
    DLE_CHECK_ARG(ld >= V && ld % 8 == 0 && ld_d >= V && ld_d % 8 == 0 && (reinterpret_cast<uintptr_t>(logits) & 15) == 0 &&
                  (reinterpret_cast<uintptr_t>(dlogits) & 15) == 0);
    if (rows == 0) return DLE_OK;
    softmax_ce_bwd_kernel<<<ce_grid(rows), CE_THREADS, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
        reinterpret_cast<const bf16*>(logits), reinterpret_cast<const long long*>(labels), lse, grad_scale, reinterpret_cast<bf16*>(dlogits),
        rows, V, ld, ld_d, ignore_index);
    DLE_LAUNCH_CHECK();
    return DLE_OK;
}
