// Shared device helpers for the sm_90a kernels: mbarrier, TMA and wgmma PTX wrappers,
// counter-based RNG for dropout, bf16 packing, tanh-GELU.  Written for
// -gencode arch=compute_90a,code=sm_90a only.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#define DLE_OK 0
#define DLE_ERR_INVALID (-22)   /* EINVAL-style: bad shape / alignment / null pointer  */
#define DLE_ERR_CUDA (-5)       /* launch / driver failure (cudaGetLastError != success) */
#define DLE_ERR_NOSYS (-38)     /* feature not compiled in                              */

#define DLE_CHECK_ARG(cond) do { if (!(cond)) return DLE_ERR_INVALID; } while (0)
#define DLE_LAUNCH_CHECK() do { if (cudaGetLastError() != cudaSuccess) return DLE_ERR_CUDA; } while (0)

namespace dle {

typedef __nv_bfloat16 bf16;
typedef __nv_bfloat162 bf162;

// ---------------------------------------------------------------------------------------------
// generic
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ uint32_t lane_id() { return threadIdx.x & 31; }
__device__ __forceinline__ bool elect_one() {
    uint32_t pred = 0;
    asm volatile("{\n.reg .pred p;\nelect.sync _|p, 0xffffffff;\nselp.u32 %0, 1, 0, p;\n}" : "=r"(pred));
    return pred != 0;
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
// One halving step of warp_column_sums32.  HALF is a template parameter so that every index into v is a compile-time constant:
// nvcc does not fully unroll a loop over `half >>= 1`, and one run-time index into v puts the whole array, and every epilogue
// row that flows into it, on the stack.
template <int HALF> __device__ __forceinline__ void column_sums_halve(float (&v)[32], int lane) {
    const bool hi = (lane & HALF) != 0;
#pragma unroll
    for (int i = 0; i < HALF; ++i) {
        const float send = hi ? v[i] : v[i + HALF];
        const float keep = hi ? v[i + HALF] : v[i];
        v[i] = keep + __shfl_xor_sync(0xffffffffu, send, HALF);
    }
}
// Column sums of a 32x32 tile held one ROW per lane (v[c] = element (lane, c)): recursive halving, 31 shuffles + 31 adds.
// On return lane l holds the sum over the 32 rows of COLUMN l.
__device__ __forceinline__ float warp_column_sums32(float (&v)[32], int lane) {
    column_sums_halve<16>(v, lane);
    column_sums_halve<8>(v, lane);
    column_sums_halve<4>(v, lane);
    column_sums_halve<2>(v, lane);
    column_sums_halve<1>(v, lane);
    return v[0];
}
__device__ __forceinline__ uint32_t pack_bf16(float lo, float hi) {
    bf162 t = __floats2bfloat162_rn(lo, hi);
    return *reinterpret_cast<uint32_t*>(&t);
}
__device__ __forceinline__ float2 unpack_bf16(uint32_t u) {
    bf162 t = *reinterpret_cast<bf162*>(&u);
    return __bfloat1622float2(t);
}

// ---------------------------------------------------------------------------------------------
// two-lane fp32 helpers (kept as pairs so the GELU / dropout code reads the same on every architecture) and byte permute
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void ffma2(float& d0, float& d1, float a0, float a1, float b0, float b1, float c0, float c1) {
    d0 = fmaf(a0, b0, c0); d1 = fmaf(a1, b1, c1);
}
__device__ __forceinline__ void fmul2(float& d0, float& d1, float a0, float a1, float b0, float b1) { d0 = a0 * b0; d1 = a1 * b1; }
__device__ __forceinline__ void fadd2(float& d0, float& d1, float a0, float a1, float b0, float b1) { d0 = a0 + b0; d1 = a1 + b1; }
__device__ __forceinline__ uint32_t prmt(uint32_t a, uint32_t b, uint32_t sel) {
    uint32_t r;
    asm("prmt.b32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(sel));
    return r;
}

// ---------------------------------------------------------------------------------------------
// math: tanh-GELU (reference modeling.py:121-122, approximate=True == tanh form)
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float tanh_fast(float x) {
    float y;
    asm("tanh.approx.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
__device__ __forceinline__ float gelu_tanh(float x) {
    const float c = 0.7978845608028654f;
    float t = tanh_fast(c * (x + 0.044715f * x * x * x));
    return 0.5f * x * (1.0f + t);
}
// two lanes at a time: 0.5 x (1 + tanh(c x (1 + 0.044715 x^2)))
__device__ __forceinline__ void gelu_tanh2(float x0, float x1, float& y0, float& y1) {
    const float c0 = 0.7978845608028654f, c1 = 0.7978845608028654f * 0.044715f;
    float s0, s1, a0, a1, h0, h1;
    fmul2(s0, s1, x0, x1, x0, x1);
    ffma2(s0, s1, s0, s1, c1, c1, c0, c0);
    fmul2(a0, a1, x0, x1, s0, s1);
    const float t0 = tanh_fast(a0), t1 = tanh_fast(a1);
    fmul2(h0, h1, x0, x1, 0.5f, 0.5f);
    ffma2(y0, y1, h0, h1, t0, t1, h0, h1);
}
// d/dx of the above for two lanes: 0.5 (1 + t) + 0.5 x (1 - t^2) c (1 + 3 * 0.044715 x^2),  t = tanh(c x (1 + 0.044715 x^2))
__device__ __forceinline__ void gelu_tanh_grad2(float x0, float x1, float& y0, float& y1) {
    const float c0 = 0.7978845608028654f, c1 = 0.7978845608028654f * 0.044715f, c3 = 3.0f * 0.7978845608028654f * 0.044715f;
    float s0, s1, i0, i1, a0, a1, d0, d1, q0, q1, h0, h1, r0, r1, g0, g1;
    fmul2(s0, s1, x0, x1, x0, x1);
    ffma2(i0, i1, s0, s1, c1, c1, c0, c0);
    fmul2(a0, a1, x0, x1, i0, i1);
    const float t0 = tanh_fast(a0), t1 = tanh_fast(a1);
    ffma2(d0, d1, -t0, -t1, t0, t1, 1.0f, 1.0f);            // 1 - t^2
    ffma2(q0, q1, s0, s1, c3, c3, c0, c0);                  // c (1 + 3 * 0.044715 x^2)
    fmul2(h0, h1, x0, x1, 0.5f, 0.5f);
    fmul2(r0, r1, h0, h1, d0, d1);
    ffma2(g0, g1, t0, t1, 0.5f, 0.5f, 0.5f, 0.5f);          // 0.5 (1 + t)
    ffma2(y0, y1, r0, r1, q0, q1, g0, g1);
}
__device__ __forceinline__ float gelu_tanh_grad(float x) {
    const float c = 0.7978845608028654f;
    float x2 = x * x;
    float t = tanh_fast(c * (x + 0.044715f * x * x2));
    return 0.5f * (1.0f + t) + 0.5f * x * (1.0f - t * t) * c * (1.0f + 3.0f * 0.044715f * x2);
}

// ---------------------------------------------------------------------------------------------
// Philox4x32-7: counter-based RNG, so forward and backward regenerate identical dropout masks
// from (seed, stream, element-group index) with no mask tensor in HBM.
// One call -> four 32-bit words -> (LCG expansion) -> keep decisions for 32 consecutive elements.
// ---------------------------------------------------------------------------------------------
template <int ROUNDS>
__device__ __forceinline__ uint4 philox4x32(uint4 ctr, uint2 key) {
    const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
#pragma unroll
    for (int r = 0; r < ROUNDS; ++r) {
        uint32_t hi0 = __umulhi(M0, ctr.x), lo0 = M0 * ctr.x;
        uint32_t hi1 = __umulhi(M1, ctr.z), lo1 = M1 * ctr.z;
        ctr = make_uint4(hi1 ^ ctr.y ^ key.x, lo1, hi0 ^ ctr.w ^ key.y, lo0);
        key.x += W0; key.y += W1;
    }
    return ctr;
}
// 32 keep-bits for the 32 consecutive elements of group `group32` (element index >> 5): ONE Philox4x32-7 call gives four
// independent 32-bit words; each word seeds a 32-bit LCG (x <- x*747796405 + 2891336453, PCG's multiplier/increment) that is
// stepped 7 times, and the top 16 bits of each state are compared with the 16-bit threshold.  The keyed, Crush-resistant
// generator decorrelates groups; inside a group the LCG's high bits are more than adequate for Bernoulli(p) decisions.
// Cost ~1.75 (Philox, amortised) + 3 instructions per element instead of ~10.
template <int ROUNDS = 7>
__device__ __forceinline__ uint32_t dropout_keep32(uint64_t seed, uint32_t stream, uint64_t group32, uint32_t thresh16) {
    const uint4 r = philox4x32<ROUNDS>(make_uint4((uint32_t)group32, (uint32_t)(group32 >> 32), stream, 0x5eed32u),
                                       make_uint2((uint32_t)seed, (uint32_t)(seed >> 32)));
    const uint32_t t = thresh16 << 16;
    uint32_t x[4] = {r.x, r.y, r.z, r.w};
    uint32_t m = 0;
#pragma unroll
    for (int w = 0; w < 4; ++w) {
        uint32_t s = x[w];
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            m |= (s >= t ? 1u : 0u) << (w * 8 + k);
            s = s * 747796405u + 2891336453u;
        }
    }
    return m;
}
// The same decisions for ONE byte of the group: bits [8*w, 8*w+8) of dropout_keep32(...), i.e. the keep bits of the 8 consecutive
// elements starting at (group32 << 5) + 8*w.  For kernels whose threads own 8 elements (LayerNorm, embedding): the Philox block is
// still needed in full, but only one of its four words is expanded (8 LCG steps instead of 32).
template <int ROUNDS = 7>
__device__ __forceinline__ uint32_t dropout_keep8(uint64_t seed, uint32_t stream, uint64_t group32, int w, uint32_t thresh16) {
    const uint4 r = philox4x32<ROUNDS>(make_uint4((uint32_t)group32, (uint32_t)(group32 >> 32), stream, 0x5eed32u),
                                       make_uint2((uint32_t)seed, (uint32_t)(seed >> 32)));
    const uint32_t t = thresh16 << 16;
    uint32_t s = (w == 0) ? r.x : (w == 1) ? r.y : (w == 2) ? r.z : r.w;
    uint32_t m = 0;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        m |= (s >= t ? 1u : 0u) << k;
        s = s * 747796405u + 2891336453u;
    }
    return m;
}
__host__ __device__ __forceinline__ uint32_t dropout_thresh16(float p) {
    float t = p * 65536.0f + 0.5f;
    return t <= 0.f ? 0u : (t >= 65535.f ? 65535u : (uint32_t)t);
}

// ---------------------------------------------------------------------------------------------
// dropout seeds under CUDA graphs: the host seed of a call site is frozen into a captured graph, so every dropout kernel also
// takes an optional DEVICE counter (`seed_dev`, bumped once per training step by dle_advance_u64); the effective seed is
// seed + *seed_dev * golden-ratio constant.  Forward and backward of one step read the same counter value.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ unsigned long long effective_seed(unsigned long long seed, const unsigned long long* seed_dev) {
    return seed_dev ? seed + __ldg(seed_dev) * 0x9E3779B97F4A7C15ull : seed;
}

// ---------------------------------------------------------------------------------------------
// Attention-probability dropout (forward and backward of the fused attention kernels): keep decisions for the 32 consecutive
// elements of group `group32`, delivered as 16 AND-masks for packed bf16x2 pairs (mask[i] covers elements 2i | 2i+1: 0xFFFF per kept
// half) -- P~ = P & mask costs one LOP3 per pair instead of a bit extract + select per element.
//   one Philox4x32-7 call -> four keyed words r_w; each is spread over four pair-words by an odd multiplier (bijective) and an
//   xor-shift (x ^ x>>16: both halfwords of the result are uniform and jointly independent); a halfword keeps its element iff its low
//   15 bits are >= t15 = round(p * 32768): (h & 0x7FFF) + (0x8000 - t15) sets bit 15 exactly then, and PRMT with sign replication
//   turns bits 15 / 31 into 0xFFFF / 0xFFFF0000.  p is therefore quantised to 1/32768; `dropout_thresh15` and the 1/(1-p) scale must
//   use the same quantised value (attn_drop_params).
// ---------------------------------------------------------------------------------------------
__host__ __device__ __forceinline__ uint32_t dropout_thresh15(float p) {
    float t = p * 32768.0f + 0.5f;
    return t <= 0.f ? 0u : (t >= 32767.f ? 32767u : (uint32_t)t);
}
// the keyed Philox block of one 32-element group, and pair-mask word i (0..15) of it
__device__ __forceinline__ uint4 attn_dropout_block(unsigned long long seed, uint32_t stream, unsigned long long group32) {
    return philox4x32<7>(make_uint4((uint32_t)group32, (uint32_t)(group32 >> 32), stream, 0xa77d20u),
                         make_uint2((uint32_t)seed, (uint32_t)(seed >> 32)));
}
__device__ __forceinline__ uint32_t attn_dropout_word(const uint4& r, int i, uint32_t k2) {
    const int w = i >> 2, k = i & 3;
    const uint32_t x = (w == 0) ? r.x : (w == 1) ? r.y : (w == 2) ? r.z : r.w;
    const uint32_t C = (k == 0) ? 0x9E3779B1u : (k == 1) ? 0x85EBCA77u : (k == 2) ? 0xC2B2AE3Du : 0x27D4EB2Fu;
    const uint32_t m = x * C;
    const uint32_t y = ((m ^ (m >> 16)) & 0x7FFF7FFFu) + k2;
    return prmt(y, 0u, 0xBB99u);
}
__device__ __forceinline__ void attn_dropout_masks16(unsigned long long seed, uint32_t stream, unsigned long long group32, uint32_t k2,
                                                     uint32_t (&mask)[16]) {
    const uint4 r = attn_dropout_block(seed, stream, group32);
#pragma unroll
    for (int i = 0; i < 16; ++i) mask[i] = attn_dropout_word(r, i, k2);
}
__host__ __device__ __forceinline__ uint32_t attn_dropout_k2(uint32_t thresh15) { return (0x8000u - thresh15) * 0x00010001u; }

// ---------------------------------------------------------------------------------------------
// mbarrier
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// Wait for the phase with the given parity.
// Watchdog: a wait that has not completed after 4 s of wall clock (kernels here last milliseconds) is a protocol bug; trap so the
// launch fails with an error instead of hanging the GPU.
// Suspend-time hint of mbarrier.try_wait: 0 = none (the hardware's default time limit per attempt), else nanoseconds.
#ifndef DLE_MBAR_HINT_NS
#define DLE_MBAR_HINT_NS 0
#endif
__device__ __forceinline__ uint32_t mbar_try_wait(uint32_t addr, uint32_t parity) {
    uint32_t ok;
#if DLE_MBAR_HINT_NS
    asm volatile(
        "{\n"
        ".reg .pred P1;\n"
        "mbarrier.try_wait.parity.shared::cta.b64 P1, [%1], %2, %3;\n"
        "selp.u32 %0, 1, 0, P1;\n"
        "}\n" : "=r"(ok) : "r"(addr), "r"(parity), "r"((uint32_t)DLE_MBAR_HINT_NS) : "memory");
#else
    asm volatile(
        "{\n"
        ".reg .pred P1;\n"
        "mbarrier.try_wait.parity.shared::cta.b64 P1, [%1], %2;\n"
        "selp.u32 %0, 1, 0, P1;\n"
        "}\n" : "=r"(ok) : "r"(addr), "r"(parity) : "memory");
#endif
    return ok;
}
__device__ __forceinline__ unsigned long long global_timer_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    const uint32_t addr = smem_u32(bar);
    if (mbar_try_wait(addr, parity)) return;
    const unsigned long long t0 = global_timer_ns();
    while (!mbar_try_wait(addr, parity)) {
        if (global_timer_ns() - t0 > 4000000000ull) __trap();
    }
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
// generic-proxy smem writes -> visible to the async proxy (TMA / wgmma operand reads)
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ---------------------------------------------------------------------------------------------
// TMA (cp.async.bulk.tensor), 2D tiles, completion on an mbarrier
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
        ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
        : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
        ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
        : "memory");
}
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* m, const void* smem_src, int c0, int c1) {
    asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
                 ::"l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(smem_src)), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void tma_store_wait_read() {
    asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
template <int N> __device__ __forceinline__ void tma_store_wait() {
    asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory");
}

// ---------------------------------------------------------------------------------------------
// warpgroup tensor-core MMA (wgmma.mma_async m64nNk16, bf16 in, fp32 accumulators in registers)
//
// Accumulator layout of one warpgroup: warp w holds rows [16w, 16w + 16); its lane l holds, for every 8-column block j, rows
// 16w + l/4 (registers 4j, 4j+1) and 16w + l/4 + 8 (4j+2, 4j+3) at columns 8j + 2(l%4) + {0,1}.  A register A operand uses the
// m16n8k16 fragment layout per warp, so two adjacent 8-column blocks of an accumulator, packed to bf16, are one k16 A fragment.
// ---------------------------------------------------------------------------------------------
// shared-memory matrix descriptor, SWIZZLE_128B: start>>4 [0,14), LBO>>4 [16,30), SBO>>4 [32,46), layout type [62,64) = 1.
// K-major operand: LBO unused, SBO = 1024 (8 rows of 128 B).  MN-major operand: LBO = stride of 64-element column chunks,
// SBO = 1024 (8 k-rows of 128 B).  The tile must sit at a 1024-byte aligned address.
__device__ __forceinline__ uint64_t make_wgmma_desc_sw128(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
    return (uint64_t)((smem_addr & 0x3FFFFu) >> 4) | ((uint64_t)(lbo_bytes >> 4) << 16) | ((uint64_t)(sbo_bytes >> 4) << 32) | (1ull << 62);
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> __device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// Pin registers that an in-flight wgmma reads or writes: the compiler must neither move their uses across the wait nor reuse them.
template <int NR> __device__ __forceinline__ void fence_regs(float (&d)[NR]) {
#pragma unroll
    for (int i = 0; i < NR; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
__device__ __forceinline__ void fence_regs(float (&d)[8][4]) {
#pragma unroll
    for (int j = 0; j < 8; ++j) asm volatile("" : "+f"(d[j][0]), "+f"(d[j][1]), "+f"(d[j][2]), "+f"(d[j][3])::"memory");
}
template <int NR> __device__ __forceinline__ void fence_regs(uint32_t (&a)[NR][2]) {
#pragma unroll
    for (int j = 0; j < NR; ++j) asm volatile("" : "+r"(a[j][0]), "+r"(a[j][1])::"memory");
}
// D (+)= A * B for one 64-row warpgroup slab, both operands in shared memory; TA / TB = 1 for an MN-major operand
template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n128k16(float (&d)[64], uint64_t desc_a, uint64_t desc_b, uint32_t scale_d) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, %67, %68;\n}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(desc_a), "l"(desc_b), "r"(scale_d), "n"(TA), "n"(TB));
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n256k16(float (&d)[128], uint64_t desc_a, uint64_t desc_b, uint32_t scale_d) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %130, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, %128, %129, p, 1, 1, %131, %132;\n}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
        : "l"(desc_a), "l"(desc_b), "r"(scale_d), "n"(TA), "n"(TB));
}
// 64 x 64 tile: d[j][0..3] is 8-column block j (layout above); A and B both in shared memory
template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n64k16(float (&d)[8][4], uint64_t desc_a, uint64_t desc_b, uint32_t scale_d) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, %35, %36;\n}\n"
        : "+f"(d[0][0]), "+f"(d[0][1]), "+f"(d[0][2]), "+f"(d[0][3]), "+f"(d[1][0]), "+f"(d[1][1]), "+f"(d[1][2]), "+f"(d[1][3]), "+f"(d[2][0]), "+f"(d[2][1]), "+f"(d[2][2]), "+f"(d[2][3]), "+f"(d[3][0]), "+f"(d[3][1]), "+f"(d[3][2]), "+f"(d[3][3]), "+f"(d[4][0]), "+f"(d[4][1]), "+f"(d[4][2]), "+f"(d[4][3]), "+f"(d[5][0]), "+f"(d[5][1]), "+f"(d[5][2]), "+f"(d[5][3]), "+f"(d[6][0]), "+f"(d[6][1]), "+f"(d[6][2]), "+f"(d[6][3]), "+f"(d[7][0]), "+f"(d[7][1]), "+f"(d[7][2]), "+f"(d[7][3])
        : "l"(desc_a), "l"(desc_b), "r"(scale_d), "n"(TA), "n"(TB));
}
// D += A * B, 64 x 64 tile with A from registers: a0..a3 = rows r | r+8 at k 0-7, then rows r | r+8 at k 8-15 of this warp's 16 rows
// (m16n8k16 layout); B in shared memory
template <int TB>
__device__ __forceinline__ void wgmma_m64n64k16_rs(float (&d)[8][4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint64_t desc_b) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %37, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, p, 1, 1, %38;\n}\n"
        : "+f"(d[0][0]), "+f"(d[0][1]), "+f"(d[0][2]), "+f"(d[0][3]), "+f"(d[1][0]), "+f"(d[1][1]), "+f"(d[1][2]), "+f"(d[1][3]), "+f"(d[2][0]), "+f"(d[2][1]), "+f"(d[2][2]), "+f"(d[2][3]), "+f"(d[3][0]), "+f"(d[3][1]), "+f"(d[3][2]), "+f"(d[3][3]), "+f"(d[4][0]), "+f"(d[4][1]), "+f"(d[4][2]), "+f"(d[4][3]), "+f"(d[5][0]), "+f"(d[5][1]), "+f"(d[5][2]), "+f"(d[5][3]), "+f"(d[6][0]), "+f"(d[6][1]), "+f"(d[6][2]), "+f"(d[6][3]), "+f"(d[7][0]), "+f"(d[7][1]), "+f"(d[7][2]), "+f"(d[7][3])
        : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "l"(desc_b), "r"(1u), "n"(TB));
}

// cp.async (LDGSTS): 16 bytes global -> shared without staging registers; groups are committed / waited per thread
__device__ __forceinline__ void cp_async16(uint32_t smem_dst, const void* gsrc) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_dst), "l"(gsrc) : "memory");
}
// copies src_bytes (0 or 16) from gsrc and zero-fills the rest of the 16 bytes: src_bytes == 0 reads nothing, but gsrc must still
// be a valid address
__device__ __forceinline__ void cp_async16_zfill(uint32_t smem_dst, const void* gsrc, uint32_t src_bytes) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_dst), "l"(gsrc), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ uint4 lds_u4(uint32_t addr) {
    uint4 r;
    asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "r"(addr));
    return r;
}

// 16-byte global store / load helpers
__device__ __forceinline__ void st_global_v4(void* p, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
    asm volatile("st.global.v4.b32 [%0], {%1, %2, %3, %4};" ::"l"(p), "r"(a), "r"(b), "r"(c), "r"(d) : "memory");
}
__device__ __forceinline__ uint4 ld_global_nc_v4(const void* p) {
    uint4 r;
    asm volatile("ld.global.nc.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
    return r;
}
__device__ __forceinline__ void red_add_v4_f32(float* p, float a, float b, float c, float d) {
    asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}

}  // namespace dle

// ---------------------------------------------------------------------------------------------
// host: TMA descriptor encode through the driver entry point (no -lcuda link dependency)
// ---------------------------------------------------------------------------------------------
namespace dle {
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
PFN_encodeTiled get_encode_tiled();
// bf16 row-major matrix [rows, cols] with leading dimension ld (elements); box = {box_cols, box_rows};
// 128B swizzle (box_cols * 2 bytes must be <= 128).
int make_tmap_bf16_2d(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols, uint64_t ld,
                      uint32_t box_cols, uint32_t box_rows);
}  // namespace dle
