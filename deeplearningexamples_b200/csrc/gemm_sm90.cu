// Dense bf16 GEMM for sm_90a: wgmma.mma_async (m64nNk16, fp32 accumulators in registers), operands staged by TMA into
// 128B-swizzled shared memory through an mbarrier ring, persistent warp-specialised CTAs: one producer warpgroup (one TMA
// warp) and two consumer warpgroups that each own 64 rows of the 128-row tile.  While the consumers run the epilogue of tile i
// the producer already streams the operands of tile i+1.
//
//   D[M,N] = A[M,K] * B[N,K]^T     (K = reduction)
//
// Either operand may be "K-major" (row-major [rows, K], the reduction dim contiguous) or
// "MN-major" (row-major [K, rows], the M/N dim contiguous) so forward (x W^T), dgrad (dy W) and
// wgrad (dy^T x) all read the tensors where they lie -- no transposed copies in HBM (wgmma reads
// MN-major bf16 operands through its transpose bits).
//
// This replaces the cuBLAS calls behind the reference's F.linear sites
// (PyTorch/LanguageModeling/BERT/modeling.py:160,345-347,395,431,553) and fuses the reference's
// separate pointwise passes (bias, tanh-GELU :121-122, dropout+residual :396-397/:432-433) into
// the epilogue.
#include <type_traits>
#include "common.cuh"
#include "../../include/dle_b200.h"

namespace dle {

constexpr int BM = 128;
constexpr int BK = 64;        // 64 bf16 = 128 B = one swizzle row
constexpr int WG_K = 16;      // k of one wgmma
// 384 threads: warpgroup 0 = producer (its first warp issues TMA), warpgroups 1 and 2 = consumers (rows 0-63 / 64-127 of the tile).
// Shared memory: the operand ring, then per consumer warpgroup a 64 x 64 fp32 accumulator staging tile (rows padded to 68 floats)
// and per consumer warp a 2 KB output staging tile + a 2 KB aux landing tile (see the epilogue below).
template <int BN> struct GemmCfg {
    static constexpr int THREADS = 384;
    static constexpr int CONSUMER_WARPS = 8;
    static constexpr int A_BYTES = BM * BK * 2;
    static constexpr int B_BYTES = BN * BK * 2;
    static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
    static constexpr int STAGES = (BN == 256) ? 3 : 4;
    static constexpr int ACC_STAGE_FLOATS_PER_ROW = 68;
    static constexpr int ACC_STAGE_BYTES = 64 * ACC_STAGE_FLOATS_PER_ROW * 4;     // per consumer warpgroup
    static constexpr int EPI_BYTES = 2 * ACC_STAGE_BYTES + CONSUMER_WARPS * 2 * 2048;
    static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + EPI_BYTES + 1024 /*align slack*/ + 256 /*barriers*/;
    static_assert(SMEM_BYTES <= 232448, "shared memory budget");
};

// wgmma shared-memory matrix descriptor, SWIZZLE_128B: start>>4 [0,14), LBO>>4 [16,30), SBO>>4 [32,46), layout type [62,64) = 1
__device__ __forceinline__ uint64_t make_wgmma_desc_sw128(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
    return (uint64_t)((smem_addr & 0x3FFFFu) >> 4) | ((uint64_t)(lbo_bytes >> 4) << 16) | ((uint64_t)(sbo_bytes >> 4) << 32) | (1ull << 62);
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> __device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
template <int NR> __device__ __forceinline__ void fence_regs(float (&d)[NR]) {
#pragma unroll
    for (int i = 0; i < NR; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// D (+)= A * B for one 64-row warpgroup slab; TA / TB = 1 for an MN-major operand
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

template <int BN, int TA, int TB>
__device__ __forceinline__ void wgmma_tile(float (&d)[BN / 2], uint64_t da, uint64_t db, uint32_t scale_d) {
    if constexpr (BN == 256) wgmma_m64n256k16<TA, TB>(d, da, db, scale_d);
    else wgmma_m64n128k16<TA, TB>(d, da, db, scale_d);
}
__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

struct GemmKernelParams {
    int M, N, K;
    int m_tiles, n_tiles, splits, kb_total;
    int epilogue;
    const bf16* bias;      // [N] or null
    const bf16* aux;       // [M, ld_aux] residual / pre-activation, or null
    void* out;             // bf16 [M, ldo] (or fp32 for DLE_EPI_ATOMIC_F32 / DLE_EPI_F32)
    bf16* out2;            // second output (pre-activation for DLE_EPI_BIAS_GELU)
    long long ldo, ld_aux, ldo2;
    float drop_scale;      // 1/(1-p)
    uint32_t drop_thresh;  // 16-bit threshold, 0 = dropout off
    uint32_t drop_stream;
    unsigned long long seed;
    const unsigned long long* seed_dev;
    float alpha;
    float* colsum_out;     // [N] fp32 or null: += column sums of the (bf16-rounded) output, e.g. the bias gradient of the layer below
};

// ----------------------------------------------------------------------------------------------
// epilogue.  The wgmma accumulator fragments are first written to a per-warpgroup fp32 staging tile; each consumer warp then
// reads back a 32-row x 32-column chunk with one ROW per lane, so the dropout mask of a 32-element RNG group, the column sums
// and the packed bf16 stores all work on whole rows.  A direct 16-byte global access per lane would touch 32 different 128-byte
// lines per warp instruction, so each warp also owns two 32 x 64 B tiles in shared memory, 16-byte units XOR-swizzled by
// (row >> 1) & 3 so that both access patterns are conflict-free:
//   out tile:  lane writes its row (4 x STS.128) -> __syncwarp -> lanes re-read as (row = it*8 + lane/4, unit = lane%4)
//              -> each ST.GLOBAL.128 covers 8 rows x 64 contiguous bytes
//   aux tile:  the residual / pre-activation operand of the chunk lands here by cp.async (row-contiguous, no registers)
//              while the accumulator chunk is staged.
// fp32 outputs (split-K atomics, logits) keep the direct path.
// ----------------------------------------------------------------------------------------------
constexpr int EPI_TILE_BYTES = 32 * 64;                 // per epilogue warp, out and aux each

__device__ __forceinline__ uint32_t epi_off(int row, int unit) { return (uint32_t)(row * 64 + ((unit ^ ((row >> 1) & 3)) << 4)); }

__device__ __forceinline__ uint4 lds_v4(uint32_t addr) {
    uint4 r;
    asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "r"(addr));
    return r;
}
__device__ __forceinline__ void sts_v4(uint32_t addr, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
    asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(a), "r"(b), "r"(c), "r"(d) : "memory");
}
__device__ __forceinline__ void cp_async_16(uint32_t smem_dst, const void* gsrc) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_dst), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }
// start the copy of rows [row_base, +32) x cols [col0, +32) of the bf16 aux matrix into this warp's aux tile
__device__ __forceinline__ void aux_prefetch(const GemmKernelParams& p, long long row_base, int col0, uint32_t aux_tile, int lane) {
#pragma unroll
    for (int it = 0; it < 4; ++it) {
        const int rr = it * 8 + (lane >> 2), cc = lane & 3;
        const long long grow = row_base + rr; const int gcol = col0 + cc * 8;
        if (grow < p.M && gcol < p.N) cp_async_16(aux_tile + epi_off(rr, cc), p.aux + grow * p.ld_aux + gcol);
    }
}
// this lane's row of the landed aux tile, still packed (4 x 8 bf16)
__device__ __forceinline__ void aux_take(uint32_t aux_tile, int lane, uint4 (&a)[4]) {
    cp_async_wait_all();
    __syncwarp();
#pragma unroll
    for (int c = 0; c < 4; ++c) a[c] = lds_v4(aux_tile + epi_off(lane, c));
    __syncwarp();
}
// this lane's row (32 floats) -> bf16 rows [row_base, +32) x cols [col0, +32) of dst, row-contiguous global stores
__device__ __forceinline__ void warp_store_rows(bf16* __restrict__ dst, long long ld, long long row_base, int col0, int M, int N,
                                                uint32_t stage, int lane, const float (&v)[32]) {
#pragma unroll
    for (int c = 0; c < 4; ++c)
        sts_v4(stage + epi_off(lane, c), pack_bf16(v[c * 8], v[c * 8 + 1]), pack_bf16(v[c * 8 + 2], v[c * 8 + 3]),
               pack_bf16(v[c * 8 + 4], v[c * 8 + 5]), pack_bf16(v[c * 8 + 6], v[c * 8 + 7]));
    __syncwarp();
    uint4 w[4];                                  // all four shared loads first: the asm statements keep program order, and a load
#pragma unroll                                   // immediately followed by its store exposes the shared-memory latency four times
    for (int it = 0; it < 4; ++it) w[it] = lds_v4(stage + epi_off(it * 8 + (lane >> 2), lane & 3));
#pragma unroll
    for (int it = 0; it < 4; ++it) {
        const int rr = it * 8 + (lane >> 2), cc = lane & 3;
        const long long grow = row_base + rr; const int gcol = col0 + cc * 8;
        if (grow < M && gcol < N) st_global_v4(dst + grow * ld + gcol, w[it].x, w[it].y, w[it].z, w[it].w);
    }
    __syncwarp();
}
__device__ __forceinline__ void unpack8(const uint4& w, float* o) {
    float2 f;
    f = unpack_bf16(w.x); o[0] = f.x; o[1] = f.y;
    f = unpack_bf16(w.y); o[2] = f.x; o[3] = f.y;
    f = unpack_bf16(w.z); o[4] = f.x; o[5] = f.y;
    f = unpack_bf16(w.w); o[6] = f.x; o[7] = f.y;
}

// one 32-row x 32-column chunk of one epilogue warp; `row` = this lane's row, row_base = first row of the warp.
// aux = this lane's row of the aux operand (packed bf16).
__device__ __forceinline__ void epilogue_chunk(const GemmKernelParams& p, const uint32_t (&acc)[32], const uint4 (&aux)[4], long long row_base,
                                               int lane, int col0, uint32_t stage, unsigned long long seed) {
    const long long row = row_base + lane;
    float v[32];
    if (p.alpha != 1.0f) {
#pragma unroll
        for (int i = 0; i < 32; ++i) v[i] = __uint_as_float(acc[i]) * p.alpha;
    } else {
#pragma unroll
        for (int i = 0; i < 32; ++i) v[i] = __uint_as_float(acc[i]);
    }
    const int ncols = min(32, p.N - col0);      // multiple of 8 (N % 8 == 0 is enforced); <= 0 for an out-of-range chunk
    if (ncols <= 0) return;                      // warp-uniform

    if (p.epilogue == DLE_EPI_ATOMIC_F32) {
        if (row < p.M) {
            float* o = reinterpret_cast<float*>(p.out) + row * p.ldo + col0;
#pragma unroll
            for (int i = 0; i < 32; i += 4)
                if (i < ncols) red_add_v4_f32(o + i, v[i], v[i + 1], v[i + 2], v[i + 3]);
        }
        return;
    }
    if (p.bias != nullptr) {                     // the same 32 values for every lane (broadcast loads); 8-byte aligned, zero beyond N
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const uint2 bw = (i * 4 < ncols) ? __ldg(reinterpret_cast<const uint2*>(p.bias + col0) + i) : make_uint2(0u, 0u);
            const float2 b0 = unpack_bf16(bw.x), b1 = unpack_bf16(bw.y);
            v[i * 4] += b0.x; v[i * 4 + 1] += b0.y; v[i * 4 + 2] += b1.x; v[i * 4 + 3] += b1.y;
        }
    }
    if (p.epilogue == DLE_EPI_F32) {
        if (row < p.M) {
            float* o = reinterpret_cast<float*>(p.out) + row * p.ldo + col0;
#pragma unroll
            for (int i = 0; i < 32; i += 4)
                if (i < ncols) *reinterpret_cast<float4*>(o + i) = make_float4(v[i], v[i + 1], v[i + 2], v[i + 3]);
        }
        return;
    }
    if (p.epilogue == DLE_EPI_BIAS_GELU) {
        // out2 = pre-activation u (needed by gelu' in backward), out = gelu(u).  gelu is evaluated on the bf16-rounded
        // pre-activation so that backward (which only has the stored bf16 u) differentiates what forward evaluated.
        warp_store_rows(p.out2, p.ldo2, row_base, col0, p.M, p.N, stage, lane, v);
#pragma unroll
        for (int i = 0; i < 32; i += 2) {
            const uint32_t u2 = pack_bf16(v[i], v[i + 1]);       // the bf16 pair just stored
            gelu_tanh2(__uint_as_float(u2 << 16), __uint_as_float(u2 & 0xFFFF0000u), v[i], v[i + 1]);
        }
    } else if (p.epilogue == DLE_EPI_BIAS_DROPOUT_RESIDUAL) {
        if (p.drop_thresh != 0) {
            const uint32_t keep = dropout_keep32(seed, p.drop_stream, (unsigned long long)(row * (long long)p.N + col0) >> 5, p.drop_thresh);
#pragma unroll
            for (int i = 0; i < 32; ++i) v[i] = ((keep >> i) & 1u) ? v[i] * p.drop_scale : 0.f;
        }
        if (p.aux != nullptr) {
#pragma unroll
            for (int c = 0; c < 4; ++c) {
                float a[8];
                unpack8(aux[c], a);
#pragma unroll
                for (int k = 0; k < 8; ++k) v[c * 8 + k] += a[k];
            }
        }
    } else if (p.epilogue == DLE_EPI_DGELU) {
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            float a[8];                                     // stored pre-activation u
            unpack8(aux[c], a);
#pragma unroll
            for (int k = 0; k < 8; k += 2) {
                float g0, g1;
                gelu_tanh_grad2(a[k], a[k + 1], g0, g1);
                fmul2(v[c * 8 + k], v[c * 8 + k + 1], v[c * 8 + k], v[c * 8 + k + 1], g0, g1);
            }
        }
    } else if (p.epilogue == DLE_EPI_ADD) {
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            float a[8];
            unpack8(aux[c], a);
#pragma unroll
            for (int k = 0; k < 8; ++k) v[c * 8 + k] += a[k];
        }
    } else if (p.epilogue == DLE_EPI_BIAS_TANH) {
#pragma unroll
        for (int i = 0; i < 32; ++i) v[i] = tanhf(v[i]);
    }
    warp_store_rows(reinterpret_cast<bf16*>(p.out), p.ldo, row_base, col0, p.M, p.N, stage, lane, v);
    if (p.colsum_out != nullptr) {
#pragma unroll
        for (int i = 0; i < 32; ++i) v[i] = (row < p.M) ? __bfloat162float(__float2bfloat16_rn(v[i])) : 0.f;
        const float cs = warp_column_sums32(v, lane);
        if (lane < ncols) atomicAdd(p.colsum_out + col0 + lane, cs);
    }
}

// ----------------------------------------------------------------------------------------------
// kernel
// ----------------------------------------------------------------------------------------------
template <int BN, bool A_MN, bool B_MN>
__global__ void __launch_bounds__(384, 1)
gemm_bf16_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                       const GemmKernelParams p) {
    using Cfg = GemmCfg<BN>;
    constexpr int NR = BN / 2;                                                 // accumulator registers per thread
    constexpr int LD = Cfg::ACC_STAGE_FLOATS_PER_ROW;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* acc_stage = smem + Cfg::STAGES * Cfg::STAGE_BYTES;               // [2 warpgroups][64][68] fp32
    uint8_t* epi_stage = acc_stage + 2 * Cfg::ACC_STAGE_BYTES;                 // [8 warps] x (out tile, aux tile)
    uint64_t* bars = reinterpret_cast<uint64_t*>(epi_stage + Cfg::CONSUMER_WARPS * 2 * EPI_TILE_BYTES);
    uint64_t* full_bar = bars;                         // [STAGES]  TMA -> consumers
    uint64_t* empty_bar = bars + Cfg::STAGES;          // [STAGES]  consumers -> TMA (one arrival per consumer warp)

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int wg = warp >> 2;

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tmap_a);
        tma_prefetch_desc(&tmap_b);
        for (int s = 0; s < Cfg::STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], Cfg::CONSUMER_WARPS); }
        fence_barrier_init();
    }
    __syncthreads();

    const int total_units = p.m_tiles * p.n_tiles * p.splits;
    const int kb_per_split = (p.kb_total + p.splits - 1) / p.splits;

    if (wg == 0) {
        // ===================== producer warpgroup: registers handed to the consumers, one warp issues TMA =====================
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;\n" ::: "memory");
        if (warp != 0) return;
        int stage = 0; uint32_t phase = 0;
        for (int unit = blockIdx.x; unit < total_units; unit += gridDim.x) {
            const int tile = unit / p.splits, split = unit - tile * p.splits;
            const int m_blk = tile / p.n_tiles, n_blk = tile - m_blk * p.n_tiles;
            const int kb0 = split * kb_per_split, kb1 = min(p.kb_total, kb0 + kb_per_split);
            for (int kb = kb0; kb < kb1; ++kb) {
                mbar_wait(&empty_bar[stage], phase ^ 1);
                if (elect_one()) {
                    mbar_expect_tx(&full_bar[stage], Cfg::STAGE_BYTES);
                    uint8_t* sa = smem + stage * Cfg::STAGE_BYTES;
                    uint8_t* sb = sa + Cfg::A_BYTES;
                    if (!A_MN) {
                        tma_load_2d(sa, &tmap_a, &full_bar[stage], kb * BK, m_blk * BM);
                    } else {
#pragma unroll
                        for (int g = 0; g < BM / 64; ++g)
                            tma_load_2d(sa + g * (BK * 128), &tmap_a, &full_bar[stage], m_blk * BM + g * 64, kb * BK);
                    }
                    if (!B_MN) {
                        tma_load_2d(sb, &tmap_b, &full_bar[stage], kb * BK, n_blk * BN);
                    } else {
#pragma unroll
                        for (int g = 0; g < BN / 64; ++g)
                            tma_load_2d(sb + g * (BK * 128), &tmap_b, &full_bar[stage], n_blk * BN + g * 64, kb * BK);
                    }
                }
                __syncwarp();
                if (++stage == Cfg::STAGES) { stage = 0; phase ^= 1; }
            }
        }
        return;
    }

    // ===================== consumer warpgroups =====================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;\n" ::: "memory");
    const int cg = wg - 1;                               // rows [cg*64, cg*64+64) of every tile
    const int cw = warp - 4;                             // consumer warp 0..7
    const int wq = warp & 3;                             // warp within the warpgroup: accumulator rows wq*16 .. +16
    const uint32_t smem_base = smem_u32(smem);
    const uint32_t stage_f32 = smem_u32(acc_stage) + cg * Cfg::ACC_STAGE_BYTES;
    const uint32_t out_tile = smem_u32(epi_stage) + cw * 2 * EPI_TILE_BYTES;
    const uint32_t aux_tile = out_tile + EPI_TILE_BYTES;
    const unsigned long long seed = (p.drop_thresh != 0u) ? effective_seed(p.seed, p.seed_dev) : 0ull;
    const bool use_aux = p.aux != nullptr && (p.epilogue == DLE_EPI_BIAS_DROPOUT_RESIDUAL || p.epilogue == DLE_EPI_DGELU ||
                                              p.epilogue == DLE_EPI_ADD);
    // epilogue chunk ownership inside the warpgroup's 64 x 64 staging tile: 32 rows x 32 columns per warp
    const int er = (wq & 1) * 32, ec = (wq >> 1) * 32;
    float d[NR];
    int stage = 0; uint32_t phase = 0;
    for (int unit = blockIdx.x; unit < total_units; unit += gridDim.x) {
        const int tile = unit / p.splits, split = unit - tile * p.splits;
        const int m_blk = tile / p.n_tiles, n_blk = tile - m_blk * p.n_tiles;
        const int kb0 = split * kb_per_split, kb1 = min(p.kb_total, kb0 + kb_per_split);
        int prev_stage = -1;
        for (int kb = kb0; kb < kb1; ++kb) {
            mbar_wait(&full_bar[stage], phase);
            const uint32_t sa = smem_base + stage * Cfg::STAGE_BYTES;
            const uint32_t sb = sa + Cfg::A_BYTES;
            fence_regs<NR>(d);
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < BK / WG_K; ++k) {
                // K-major:  rows of 128 B, 8-row groups 1024 B apart (SBO); advance 32 B per k16.
                // MN-major: k-rows of 128 B (64 m/n elements), 8-k-row groups 1024 B apart (SBO), next 64 m/n elements BK*128 B
                //           further (LBO); advance 16 k-rows = 2048 B.  This warpgroup's 64 rows start 64 rows (8 KB) in.
                const uint64_t da = A_MN ? make_wgmma_desc_sw128(sa + cg * (BK * 128) + k * (WG_K * 128), BK * 128, 1024)
                                         : make_wgmma_desc_sw128(sa + cg * (64 * 128) + k * (WG_K * 2), 16, 1024);
                const uint64_t db = B_MN ? make_wgmma_desc_sw128(sb + k * (WG_K * 128), BK * 128, 1024)
                                         : make_wgmma_desc_sw128(sb + k * (WG_K * 2), 16, 1024);
                wgmma_tile<BN, A_MN ? 1 : 0, B_MN ? 1 : 0>(d, da, db, (kb > kb0 || k > 0) ? 1u : 0u);
            }
            wgmma_commit();
            fence_regs<NR>(d);
            wgmma_wait<1>();                             // the previous k-block's MMAs have retired: its stage may be refilled
            if (prev_stage >= 0 && lane == 0) mbar_arrive(&empty_bar[prev_stage]);
            prev_stage = stage;
            if (++stage == Cfg::STAGES) { stage = 0; phase ^= 1; }
        }
        wgmma_wait<0>();
        fence_regs<NR>(d);
        if (prev_stage >= 0 && lane == 0) mbar_arrive(&empty_bar[prev_stage]);

        // ---- epilogue, 64 columns at a time: fragments -> fp32 staging -> one row per lane -> epilogue_chunk
        const long long row_base = (long long)m_blk * BM + cg * 64 + er;
        const int fr = wq * 16 + (lane >> 2), fc = 2 * (lane & 3);          // fragment row / column of this thread
#pragma unroll
        for (int cc = 0; cc < BN / 64; ++cc) {
            const int col0 = n_blk * BN + cc * 64 + ec;
            const bool live = row_base < p.M && col0 < p.N;                 // warp-uniform
            if (use_aux && live) aux_prefetch(p, row_base, col0, aux_tile, lane);
            named_bar_sync(1 + cg, 128);                                    // the previous chunk's staging reads are done
#pragma unroll
            for (int j = 0; j < 8; ++j) {                                   // 8-column groups of this 64-column chunk
                const int f = (cc * 8 + j) * 4;
                const uint32_t a0 = stage_f32 + (uint32_t)((fr * LD + j * 8 + fc) * 4);
                asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(a0), "f"(d[f]), "f"(d[f + 1]) : "memory");
                asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(a0 + 8 * LD * 4), "f"(d[f + 2]), "f"(d[f + 3]) : "memory");
            }
            named_bar_sync(1 + cg, 128);
            uint32_t r[32];
#pragma unroll
            for (int c = 0; c < 8; ++c) {
                const uint4 w = lds_v4(stage_f32 + (uint32_t)(((er + lane) * LD + ec + c * 4) * 4));
                r[c * 4] = w.x; r[c * 4 + 1] = w.y; r[c * 4 + 2] = w.z; r[c * 4 + 3] = w.w;
            }
            uint4 a[4];
            if (use_aux && live) {
                aux_take(aux_tile, lane, a);
            } else {
#pragma unroll
                for (int k = 0; k < 4; ++k) a[k] = make_uint4(0u, 0u, 0u, 0u);
            }
            if (live) epilogue_chunk(p, r, a, row_base, lane, col0, out_tile, seed);
        }
    }
}

// ----------------------------------------------------------------------------------------------
// host
// ----------------------------------------------------------------------------------------------
PFN_encodeTiled get_encode_tiled() {
    static PFN_encodeTiled fn = nullptr;
    if (fn == nullptr) {
        void* ptr = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) != cudaSuccess ||
            qres != cudaDriverEntryPointSuccess)
            return nullptr;
        fn = reinterpret_cast<PFN_encodeTiled>(ptr);
    }
    return fn;
}

int make_tmap_bf16_2d(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols, uint64_t ld,
                      uint32_t box_cols, uint32_t box_rows) {
    PFN_encodeTiled enc = get_encode_tiled();
    if (enc == nullptr) return DLE_ERR_CUDA;
    if ((reinterpret_cast<uintptr_t>(base) & 15) != 0 || (ld * 2) % 16 != 0 || box_cols * 2 > 128 || box_rows > 256)
        return DLE_ERR_INVALID;
    cuuint64_t gdim[2] = {cols, rows};
    cuuint64_t gstride[1] = {ld * 2};
    cuuint32_t box[2] = {box_cols, box_rows};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = enc(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), gdim, gstride, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS ? DLE_OK : DLE_ERR_CUDA;
}

static int num_sms() {
    static int sms[64] = {};
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev < 0 || dev >= 64) return 132;
    if (sms[dev] == 0) {
        cudaDeviceGetAttribute(&sms[dev], cudaDevAttrMultiProcessorCount, dev);
        if (sms[dev] <= 0) sms[dev] = 132;
    }
    return sms[dev];
}

template <int BN, bool A_MN, bool B_MN>
static int launch_gemm(const dle_gemm_args* a, cudaStream_t stream) {
    using Cfg = GemmCfg<BN>;
    CUtensorMap ta, tb;
    int rc;
    // K-major operand: matrix [rows, K] -> box {64 (k), rows_per_tile}; MN-major: matrix [K, rows] -> box {64 (m/n), 64 (k)}
    rc = A_MN ? make_tmap_bf16_2d(&ta, a->A, a->K, a->M, a->lda, 64, BK) : make_tmap_bf16_2d(&ta, a->A, a->M, a->K, a->lda, BK, BM);
    if (rc != DLE_OK) return rc;
    rc = B_MN ? make_tmap_bf16_2d(&tb, a->B, a->K, a->N, a->ldb, 64, BK) : make_tmap_bf16_2d(&tb, a->B, a->N, a->K, a->ldb, BK, BN);
    if (rc != DLE_OK) return rc;

    GemmKernelParams p;
    p.M = a->M; p.N = a->N; p.K = a->K;
    p.m_tiles = (a->M + BM - 1) / BM;
    p.n_tiles = (a->N + BN - 1) / BN;
    p.kb_total = (a->K + BK - 1) / BK;
    int splits = a->splits > 0 ? a->splits : 1;
    if (a->epilogue != DLE_EPI_ATOMIC_F32) splits = 1;
    if (splits > p.kb_total) splits = p.kb_total;
    // no empty split: shrink until ceil-division leaves work for the last one
    while (splits > 1 && (splits - 1) * ((p.kb_total + splits - 1) / splits) >= p.kb_total) --splits;
    p.splits = splits;
    p.epilogue = a->epilogue;
    p.bias = reinterpret_cast<const bf16*>(a->bias);
    p.aux = reinterpret_cast<const bf16*>(a->aux);
    p.out = a->out;
    p.out2 = reinterpret_cast<bf16*>(a->out2);
    p.ldo = a->ldo; p.ld_aux = a->ld_aux; p.ldo2 = a->ldo2;
    p.drop_thresh = (a->dropout_p > 0.f) ? dropout_thresh16(a->dropout_p) : 0u;
    p.drop_scale = (a->dropout_p > 0.f) ? 1.0f / (1.0f - a->dropout_p) : 1.0f;
    p.drop_stream = a->dropout_stream;
    p.seed = a->seed;
    p.seed_dev = reinterpret_cast<const unsigned long long*>(a->seed_dev);
    p.alpha = a->alpha;
    p.colsum_out = reinterpret_cast<float*>(a->colsum_out);

    auto kern = gemm_bf16_wgmma_kernel<BN, A_MN, B_MN>;
    static bool attr_set[64] = {};                      // the attribute is per device (and per template instance)
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return DLE_ERR_CUDA;
    if (!attr_set[dev]) {
        if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES) != cudaSuccess)
            return DLE_ERR_CUDA;
        attr_set[dev] = true;
    }
    const int units = p.m_tiles * p.n_tiles * p.splits;
    const int grid = units < num_sms() ? units : num_sms();
    kern<<<grid, Cfg::THREADS, Cfg::SMEM_BYTES, stream>>>(ta, tb, p);
    DLE_LAUNCH_CHECK();
    return DLE_OK;
}

}  // namespace dle

extern "C" int dle_gemm_bf16(const dle_gemm_args* a, void* stream_) {
    using namespace dle;
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    DLE_CHECK_ARG(a != nullptr && a->A != nullptr && a->B != nullptr && a->out != nullptr);
    DLE_CHECK_ARG(a->M > 0 && a->N > 0 && a->K > 0);
    // N % 8: the epilogue stores 16-byte vectors; lda/ldb % 8: TMA row strides are multiples of 16 bytes.
    // M and K are otherwise free (TMA zero-fills out-of-bounds rows/columns of partial tiles).
    DLE_CHECK_ARG(a->N % 8 == 0 && a->ldo % 8 == 0 && a->lda % 8 == 0 && a->ldb % 8 == 0);
    DLE_CHECK_ARG(a->epilogue >= 0 && a->epilogue < DLE_EPI_COUNT);
    if (a->epilogue == DLE_EPI_BIAS_DROPOUT_RESIDUAL && a->dropout_p > 0.f) DLE_CHECK_ARG(a->N % 32 == 0);   // 32-element RNG groups
    if (a->epilogue == DLE_EPI_BIAS_GELU) DLE_CHECK_ARG(a->out2 != nullptr && a->ldo2 % 8 == 0);
    if (a->epilogue == DLE_EPI_DGELU || a->epilogue == DLE_EPI_ADD) DLE_CHECK_ARG(a->aux != nullptr);
    if (a->aux != nullptr) DLE_CHECK_ARG(a->ld_aux % 8 == 0 && (reinterpret_cast<uintptr_t>(a->aux) & 15) == 0);
    // the epilogue reads the bias slice with 4- / 8-byte loads and stores 16-byte vectors
    DLE_CHECK_ARG((reinterpret_cast<uintptr_t>(a->bias) & 7) == 0 && (reinterpret_cast<uintptr_t>(a->out) & 15) == 0 &&
                  (reinterpret_cast<uintptr_t>(a->out2) & 15) == 0);
    const bool amn = a->a_layout == DLE_LAYOUT_MN, bmn = a->b_layout == DLE_LAYOUT_MN;
    // narrow-N problems (and the small-tile preference flag) take the 128-wide tile
    const bool bn128 = (a->N <= 128) || (a->tile_n == 128);
    if (bn128) {
        if (!amn && !bmn) return launch_gemm<128, false, false>(a, stream);
        if (!amn && bmn) return launch_gemm<128, false, true>(a, stream);
        if (amn && bmn) return launch_gemm<128, true, true>(a, stream);
        return launch_gemm<128, true, false>(a, stream);
    }
    if (!amn && !bmn) return launch_gemm<256, false, false>(a, stream);
    if (!amn && bmn) return launch_gemm<256, false, true>(a, stream);
    if (amn && bmn) return launch_gemm<256, true, true>(a, stream);
    return launch_gemm<256, true, false>(a, stream);
}
