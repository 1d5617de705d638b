// Multi-tensor LAMB for sm_90a: the whole optimizer step over every parameter tensor in three
// launches driven by a device-resident tensor/chunk table (built once), instead of the reference's
// ~100 launches whose tensor lists travel through 4 KB kernel-argument structs.
//
//   launch 1  grad pass   : sum g^2 over all tensors (fp32 lanes -> double atomics), non-finite
//                           detection; the last CTA to finish derives found_inf, the clip factor,
//                           inv_scale, increments each group's step and computes bias corrections.
//   launch 2  stage 1     : m,v update; per-tensor sum p^2 and sum u^2 (u is NOT stored)
//   launch 3  stage 2     : recompute u from (m_new, v_new, p) -- bit-identical to stage 1 --
//                           apply p -= lr * |p|/|u| * u, write the bf16 model copy.
//
// HBM bytes per parameter (bf16 grad, fp32 p/m/v, bf16 model copy): 2 | 2+12+8 | 12+4+2 = 42 B
// (algorithmic minimum 28 B; the reference moves ~56 B).  Math follows
// lamb_amp_opt/csrc/multi_tensor_lamb.cu:67-79,121-157,274-282 and fused_lamb.py:148-204.
#include "common.cuh"
#include "../../include/dle_b200.h"

namespace dle {

constexpr int LAMB_THREADS = 512;
constexpr int LAMB_CHUNK = 16384;          // elements per work item

struct LambTensorDev {
    void* g; float* p; float* m; float* v; void* pm;
    long long n;
    int group; int pad;
};
struct LambGroupDev {
    const float* lr; int* step;
    float beta1, beta2, eps, wd;
    int bias_correction, grad_averaging;
    float bc1, bc2;                          // written by the grad pass each step
    float beta3; int pad;
};
struct LambState {                           // device scalars shared by the three launches
    double gsq;                              // running sum of g^2 (self-resetting)
    unsigned int ticket; unsigned int nonfinite;
    float gnorm, found_inf, clip, inv_scale;
};
struct LambPlan {                            // host-side handle
    LambTensorDev* tensors; LambGroupDev* groups; int2* chunks; LambState* state;
    double* psq; double* usq;                // [n_tensors] each
    void* block; size_t block_bytes;
    int n_tensors, n_groups, n_chunks, grad_dtype;
    long long total_numel;
    // pinned staging for dle_lamb_plan_update: a ring of LAMB_EAGER_SLOTS slots (one event each: a slot is rewritten only after the
    // copy that read it has run) plus LAMB_CAPTURE_SLOTS slots that are handed out once each to updates issued under CUDA-graph
    // capture (the captured copy node re-reads its slot on every replay, so such a slot is never reused).  Allocated at plan creation:
    // nothing on the per-step path allocates or synchronises.
    LambTensorDev* host_stage = nullptr; long long* stage_numel = nullptr;
    cudaEvent_t stage_event[8] = {}; bool stage_used[8] = {};
    int next_slot = 0, next_capture_slot = 0;
};
constexpr int LAMB_EAGER_SLOTS = 8, LAMB_CAPTURE_SLOTS = 4;

__device__ __forceinline__ float block_reduce_sum(float v, float* sh) {
    v = warp_sum(v);
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
    __syncthreads();
    if (l == 0) sh[w] = v;
    __syncthreads();
    float r = (threadIdx.x < (blockDim.x >> 5)) ? sh[threadIdx.x] : 0.f;
    if (w == 0) r = warp_sum(r);
    return r;                                 // valid in warp 0
}

template <typename G> __device__ __forceinline__ void load4(const G* p, float (&o)[4]);
template <> __device__ __forceinline__ void load4<float>(const float* p, float (&o)[4]) {
    float4 t = *reinterpret_cast<const float4*>(p); o[0] = t.x; o[1] = t.y; o[2] = t.z; o[3] = t.w;
}
template <> __device__ __forceinline__ void load4<bf16>(const bf16* p, float (&o)[4]) {
    uint2 t = *reinterpret_cast<const uint2*>(p);
    float2 a = unpack_bf16(t.x), b = unpack_bf16(t.y); o[0] = a.x; o[1] = a.y; o[2] = b.x; o[3] = b.y;
}
__device__ __forceinline__ float to_f(float x) { return x; }
__device__ __forceinline__ float to_f(bf16 x) { return __bfloat162float(x); }

// ---------------------------------------------------------------------------------------------
// launch 1: global gradient norm + found_inf + per-step scalars
// ---------------------------------------------------------------------------------------------
template <typename G>
__global__ void __launch_bounds__(LAMB_THREADS)
lamb_grad_pass(const LambTensorDev* __restrict__ tensors, const int2* __restrict__ chunks, int n_chunks,
               LambGroupDev* groups, int n_groups, LambState* st, double* psq, double* usq, int n_tensors,
               const float* scale_ptr, float max_grad_norm, float clip_eps, int advance_step,
               float* found_inf_out, float* gnorm_out) {
    __shared__ float sh[32];
    float acc = 0.f;
    for (int c = blockIdx.x; c < n_chunks; c += gridDim.x) {
        const int2 ch = chunks[c];
        const LambTensorDev t = tensors[ch.x];
        const long long off = (long long)ch.y * LAMB_CHUNK;
        const int n = (int)min((long long)LAMB_CHUNK, t.n - off);
        const G* g = reinterpret_cast<const G*>(t.g) + off;
        if ((reinterpret_cast<uintptr_t>(g) & (4 * sizeof(G) - 1)) == 0 && (n & 3) == 0) {
            for (int i = threadIdx.x * 4; i < n; i += LAMB_THREADS * 4) {
                float x[4]; load4<G>(g + i, x);
                acc += x[0] * x[0] + x[1] * x[1] + x[2] * x[2] + x[3] * x[3];
            }
        } else {
            for (int i = threadIdx.x; i < n; i += LAMB_THREADS) { float x = to_f(g[i]); acc += x * x; }
        }
    }
    float tot = block_reduce_sum(acc, sh);
    __shared__ bool is_last;
    if (threadIdx.x == 0) {
        if (!isfinite(tot)) atomicOr(&st->nonfinite, 1u);
        else atomicAdd(&st->gsq, (double)tot);
        __threadfence();
        unsigned int tk = atomicAdd(&st->ticket, 1u);
        is_last = (tk == gridDim.x - 1);
    }
    __syncthreads();
    if (!is_last) return;
    // ---- last CTA: finalise the step scalars (fused_lamb.py:148-165,201-204; multi_tensor_lamb.cu:67-77)
    __threadfence();
    for (int i = threadIdx.x; i < n_tensors; i += blockDim.x) { psq[i] = 0.0; usq[i] = 0.0; }
    if (threadIdx.x == 0) {
        const double gsq = *reinterpret_cast<volatile double*>(&st->gsq);
        const unsigned int bad = *reinterpret_cast<volatile unsigned int*>(&st->nonfinite);
        float gnorm = (float)sqrt(gsq);
        const bool inf = (bad != 0u) || !isfinite(gnorm);
        if (inf) gnorm = __int_as_float(0x7f800000);
        const float scale = scale_ptr ? *scale_ptr : 1.0f;
        const float inv_scale = (float)(1.0 / (double)scale);
        const float max_norm = max_grad_norm * scale;
        st->gnorm = gnorm;
        st->found_inf = inf ? 1.0f : 0.0f;
        // LAMB (multi_tensor_lamb.cu:77): gnorm > max ? gnorm/max : 1.   SQuAD GradientClipper (run_squad.py:721-724):
        // coef = max/(gnorm + 1e-6), applied when < 1.  clip_eps selects between them; max_grad_norm <= 0 disables clipping.
        st->clip = (max_grad_norm > 0.f && (gnorm + clip_eps * scale) > max_norm) ? (gnorm + clip_eps * scale) / max_norm : 1.0f;
        st->inv_scale = inv_scale;
        if (found_inf_out) *found_inf_out = inf ? 1.0f : 0.0f;
        if (gnorm_out) *gnorm_out = gnorm;
        if (advance_step) {
            for (int gi = 0; gi < n_groups; ++gi) {
                LambGroupDev& G_ = groups[gi];
                int step = *G_.step;
                if (!inf) { step += 1; *G_.step = step; }
                if (G_.bias_correction) {
                    G_.bc1 = (float)(1.0 - pow((double)G_.beta1, (double)step));
                    G_.bc2 = (float)(1.0 - pow((double)G_.beta2, (double)step));
                } else { G_.bc1 = 1.0f; G_.bc2 = 1.0f; }
                G_.beta3 = G_.grad_averaging ? 1.0f - G_.beta1 : 1.0f;
            }
        }
        st->gsq = 0.0; st->nonfinite = 0u; st->ticket = 0u;     // self-reset for the next step
    }
}

// ---------------------------------------------------------------------------------------------
// shared element math
// ---------------------------------------------------------------------------------------------
struct LambHyper { float b1, b2, b3, bc1, bc2, eps, wd, clip, inv_scale; int adam_w; };

__device__ __forceinline__ void lamb_moments(const LambHyper& h, float g, float p, float& m, float& v) {
    float sg = (g * h.inv_scale) / h.clip;
    if (!h.adam_w) sg = sg + h.wd * p;                       // MOMENT_MODE_0 (L2)
    m = m * h.b1 + h.b3 * sg;
    v = v * h.b2 + (1.0f - h.b2) * sg * sg;
}
__device__ __forceinline__ float lamb_update(const LambHyper& h, float p, float m, float v) {
    float mu = m / h.bc1, vu = v / h.bc2;
    float u = mu / (sqrtf(vu) + h.eps);
    if (h.adam_w) u = u + h.wd * p;                          // MOMENT_MODE_1 (decoupled decay)
    return u;
}

// ---------------------------------------------------------------------------------------------
// launch 2: stage 1
// ---------------------------------------------------------------------------------------------
template <typename G>
__global__ void __launch_bounds__(LAMB_THREADS)
lamb_stage1(const LambTensorDev* __restrict__ tensors, const int2* __restrict__ chunks, int n_chunks,
            const LambGroupDev* __restrict__ groups, const LambState* __restrict__ st, double* psq, double* usq,
            int adam_w) {
    if (st->found_inf != 0.0f) return;                        // noop protocol (multi_tensor_lamb.cu:63-65)
    __shared__ float sh[32];
    for (int c = blockIdx.x; c < n_chunks; c += gridDim.x) {
        const int2 ch = chunks[c];
        const LambTensorDev t = tensors[ch.x];
        const LambGroupDev G_ = groups[t.group];
        LambHyper h{G_.beta1, G_.beta2, G_.beta3, G_.bc1, G_.bc2, G_.eps, G_.wd, st->clip, st->inv_scale, adam_w};
        const long long off = (long long)ch.y * LAMB_CHUNK;
        const int n = (int)min((long long)LAMB_CHUNK, t.n - off);
        const G* g = reinterpret_cast<const G*>(t.g) + off;
        float* p = t.p + off; float* m = t.m + off; float* v = t.v + off;
        float ps = 0.f, us = 0.f;
        const bool vec = ((reinterpret_cast<uintptr_t>(g) & (4 * sizeof(G) - 1)) == 0) &&
                         (((reinterpret_cast<uintptr_t>(p) | reinterpret_cast<uintptr_t>(m) | reinterpret_cast<uintptr_t>(v)) & 15) == 0) &&
                         ((n & 3) == 0);
        if (vec) {
            for (int i = threadIdx.x * 4; i < n; i += LAMB_THREADS * 4) {
                float gg[4]; load4<G>(g + i, gg);
                float4 pp = *reinterpret_cast<const float4*>(p + i);
                float4 mm = *reinterpret_cast<const float4*>(m + i);
                float4 vv = *reinterpret_cast<const float4*>(v + i);
                float pa[4] = {pp.x, pp.y, pp.z, pp.w}, ma[4] = {mm.x, mm.y, mm.z, mm.w}, va[4] = {vv.x, vv.y, vv.z, vv.w};
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    lamb_moments(h, gg[k], pa[k], ma[k], va[k]);
                    float u = lamb_update(h, pa[k], ma[k], va[k]);
                    ps += pa[k] * pa[k]; us += u * u;
                }
                *reinterpret_cast<float4*>(m + i) = make_float4(ma[0], ma[1], ma[2], ma[3]);
                *reinterpret_cast<float4*>(v + i) = make_float4(va[0], va[1], va[2], va[3]);
            }
        } else {
            for (int i = threadIdx.x; i < n; i += LAMB_THREADS) {
                float gg = to_f(g[i]), pp = p[i], mm = m[i], vv = v[i];
                lamb_moments(h, gg, pp, mm, vv);
                float u = lamb_update(h, pp, mm, vv);
                ps += pp * pp; us += u * u;
                m[i] = mm; v[i] = vv;
            }
        }
        float pt = block_reduce_sum(ps, sh);
        float ut = block_reduce_sum(us, sh);
        if (threadIdx.x == 0) { atomicAdd(&psq[ch.x], (double)pt); atomicAdd(&usq[ch.x], (double)ut); }
    }
}

// ---------------------------------------------------------------------------------------------
// launch 3: stage 2
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(LAMB_THREADS)
lamb_stage2(const LambTensorDev* __restrict__ tensors, const int2* __restrict__ chunks, int n_chunks,
            const LambGroupDev* __restrict__ groups, const LambState* __restrict__ st, const double* __restrict__ psq,
            const double* __restrict__ usq, int adam_w, int use_nvlamb, float* norms_out, int n_tensors) {
    if (st->found_inf != 0.0f) return;
    for (int c = blockIdx.x; c < n_chunks; c += gridDim.x) {
        const int2 ch = chunks[c];
        const LambTensorDev t = tensors[ch.x];
        const LambGroupDev G_ = groups[t.group];
        LambHyper h{G_.beta1, G_.beta2, G_.beta3, G_.bc1, G_.bc2, G_.eps, G_.wd, st->clip, st->inv_scale, adam_w};
        const float lr = *G_.lr;
        const float pn = (float)sqrt(psq[ch.x]), un = (float)sqrt(usq[ch.x]);
        float ratio = lr;                                        // multi_tensor_lamb.cu:274-282
        if (use_nvlamb || G_.wd != 0.0f) ratio = (un != 0.0f && pn != 0.0f) ? lr * (pn / un) : lr;
        if (norms_out && ch.y == 0 && threadIdx.x == 0) { norms_out[ch.x] = pn; norms_out[n_tensors + ch.x] = un; }
        const long long off = (long long)ch.y * LAMB_CHUNK;
        const int n = (int)min((long long)LAMB_CHUNK, t.n - off);
        float* p = t.p + off; const float* m = t.m + off; const float* v = t.v + off;
        bf16* pm = t.pm ? reinterpret_cast<bf16*>(t.pm) + off : nullptr;
        const bool vec = (((reinterpret_cast<uintptr_t>(p) | reinterpret_cast<uintptr_t>(m) | reinterpret_cast<uintptr_t>(v)) & 15) == 0) &&
                         ((reinterpret_cast<uintptr_t>(pm) & 7) == 0) && ((n & 3) == 0);
        if (vec) {
            for (int i = threadIdx.x * 4; i < n; i += LAMB_THREADS * 4) {
                float4 pp = *reinterpret_cast<const float4*>(p + i);
                float4 mm = *reinterpret_cast<const float4*>(m + i);
                float4 vv = *reinterpret_cast<const float4*>(v + i);
                pp.x -= ratio * lamb_update(h, pp.x, mm.x, vv.x);
                pp.y -= ratio * lamb_update(h, pp.y, mm.y, vv.y);
                pp.z -= ratio * lamb_update(h, pp.z, mm.z, vv.z);
                pp.w -= ratio * lamb_update(h, pp.w, mm.w, vv.w);
                *reinterpret_cast<float4*>(p + i) = pp;
                if (pm) *reinterpret_cast<uint2*>(pm + i) = make_uint2(pack_bf16(pp.x, pp.y), pack_bf16(pp.z, pp.w));
            }
        } else {
            for (int i = threadIdx.x; i < n; i += LAMB_THREADS) {
                float pp = p[i];
                pp -= ratio * lamb_update(h, pp, m[i], v[i]);
                p[i] = pp;
                if (pm) pm[i] = __float2bfloat16_rn(pp);
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------
// multi-tensor Adam / AdamW on the same tables: after the grad pass (norm, found_inf, step++, bias corrections) ONE fused
// pass updates m, v, p and the bf16 model copy (no trust ratio => no second sweep): 2 + 14 + 14 = 30 B/param.
// replaces apex.optimizers.FusedAdam + the amp_C l2norm/scale clipper of run_squad.py:703-724,969-975 (apex is not vendored:
// the arithmetic is the published Adam/AdamW update, anchored on those call sites).
// ---------------------------------------------------------------------------------------------
template <typename G>
__global__ void __launch_bounds__(LAMB_THREADS)
adam_apply(const LambTensorDev* __restrict__ tensors, const int2* __restrict__ chunks, int n_chunks,
           const LambGroupDev* __restrict__ groups, const LambState* __restrict__ st, int adam_w) {
    if (st->found_inf != 0.0f) return;
    for (int c = blockIdx.x; c < n_chunks; c += gridDim.x) {
        const int2 ch = chunks[c];
        const LambTensorDev t = tensors[ch.x];
        const LambGroupDev G_ = groups[t.group];
        LambHyper h{G_.beta1, G_.beta2, 1.0f - G_.beta1, G_.bc1, G_.bc2, G_.eps, G_.wd, st->clip, st->inv_scale, adam_w};
        const float lr = *G_.lr;
        const long long off = (long long)ch.y * LAMB_CHUNK;
        const int n = (int)min((long long)LAMB_CHUNK, t.n - off);
        const G* g = reinterpret_cast<const G*>(t.g) + off;
        float* p = t.p + off; float* m = t.m + off; float* v = t.v + off;
        bf16* pm = t.pm ? reinterpret_cast<bf16*>(t.pm) + off : nullptr;
        const bool vec = ((reinterpret_cast<uintptr_t>(g) & (4 * sizeof(G) - 1)) == 0) &&
                         (((reinterpret_cast<uintptr_t>(p) | reinterpret_cast<uintptr_t>(m) | reinterpret_cast<uintptr_t>(v)) & 15) == 0) &&
                         ((reinterpret_cast<uintptr_t>(pm) & 7) == 0) && ((n & 3) == 0);
        if (vec) {
            for (int i = threadIdx.x * 4; i < n; i += LAMB_THREADS * 4) {
                float gg[4]; load4<G>(g + i, gg);
                float4 pp = *reinterpret_cast<const float4*>(p + i);
                float4 mm = *reinterpret_cast<const float4*>(m + i);
                float4 vv = *reinterpret_cast<const float4*>(v + i);
                float pa[4] = {pp.x, pp.y, pp.z, pp.w}, ma[4] = {mm.x, mm.y, mm.z, mm.w}, va[4] = {vv.x, vv.y, vv.z, vv.w};
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    lamb_moments(h, gg[k], pa[k], ma[k], va[k]);
                    pa[k] -= lr * lamb_update(h, pa[k], ma[k], va[k]);
                }
                *reinterpret_cast<float4*>(p + i) = make_float4(pa[0], pa[1], pa[2], pa[3]);
                *reinterpret_cast<float4*>(m + i) = make_float4(ma[0], ma[1], ma[2], ma[3]);
                *reinterpret_cast<float4*>(v + i) = make_float4(va[0], va[1], va[2], va[3]);
                if (pm) *reinterpret_cast<uint2*>(pm + i) = make_uint2(pack_bf16(pa[0], pa[1]), pack_bf16(pa[2], pa[3]));
            }
        } else {
            for (int i = threadIdx.x; i < n; i += LAMB_THREADS) {
                float gg = to_f(g[i]), pp = p[i], mm = m[i], vv = v[i];
                lamb_moments(h, gg, pp, mm, vv);
                pp -= lr * lamb_update(h, pp, mm, vv);
                p[i] = pp; m[i] = mm; v[i] = vv;
                if (pm) pm[i] = __float2bfloat16_rn(pp);
            }
        }
    }
}

static int lamb_grid(int n_chunks) {
    int dev = 0, sms = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    int g = sms * 4;                                            // 4 x 512-thread CTAs resident per SM
    return n_chunks < g ? (n_chunks > 0 ? n_chunks : 1) : g;
}

}  // namespace dle

using namespace dle;

extern "C" int dle_lamb_plan_create(const dle_lamb_tensor* ht, int32_t n_tensors, const dle_lamb_group* hg,
                                    int32_t n_groups, int32_t grad_dtype, void** plan_out) {
    DLE_CHECK_ARG(ht && hg && plan_out && n_tensors > 0 && n_groups > 0);
    DLE_CHECK_ARG(grad_dtype == DLE_DTYPE_F32 || grad_dtype == DLE_DTYPE_BF16);
    long long n_chunks = 0, total = 0;
    for (int i = 0; i < n_tensors; ++i) {
        DLE_CHECK_ARG(ht[i].grad && ht[i].param && ht[i].exp_avg && ht[i].exp_avg_sq && ht[i].numel > 0);
        DLE_CHECK_ARG(ht[i].group >= 0 && ht[i].group < n_groups);
        n_chunks += (ht[i].numel + LAMB_CHUNK - 1) / LAMB_CHUNK;
        total += ht[i].numel;
    }
    DLE_CHECK_ARG(n_chunks < (1ll << 30));
    auto up = [](size_t x) { return (x + 255) & ~size_t(255); };
    const size_t o_t = 0, o_g = o_t + up(sizeof(LambTensorDev) * n_tensors), o_c = o_g + up(sizeof(LambGroupDev) * n_groups),
                 o_s = o_c + up(sizeof(int2) * n_chunks), o_p = o_s + up(sizeof(LambState)),
                 o_u = o_p + up(sizeof(double) * n_tensors), bytes = o_u + up(sizeof(double) * n_tensors);
    uint8_t* host = static_cast<uint8_t*>(calloc(1, bytes));
    if (!host) return DLE_ERR_CUDA;
    LambTensorDev* t = reinterpret_cast<LambTensorDev*>(host + o_t);
    LambGroupDev* g = reinterpret_cast<LambGroupDev*>(host + o_g);
    int2* c = reinterpret_cast<int2*>(host + o_c);
    long long ci = 0;
    for (int i = 0; i < n_tensors; ++i) {
        t[i] = LambTensorDev{ht[i].grad, ht[i].param, ht[i].exp_avg, ht[i].exp_avg_sq, ht[i].model_param, ht[i].numel, ht[i].group, 0};
        const int nc = (int)((ht[i].numel + LAMB_CHUNK - 1) / LAMB_CHUNK);
        for (int k = 0; k < nc; ++k) c[ci++] = make_int2(i, k);
    }
    for (int i = 0; i < n_groups; ++i) {
        DLE_CHECK_ARG(hg[i].lr && hg[i].step);
        g[i] = LambGroupDev{hg[i].lr, hg[i].step, hg[i].beta1, hg[i].beta2, hg[i].eps, hg[i].weight_decay,
                            hg[i].bias_correction, hg[i].grad_averaging, 1.0f, 1.0f,
                            hg[i].grad_averaging ? 1.0f - hg[i].beta1 : 1.0f, 0};
    }
    void* dev = nullptr;
    if (cudaMalloc(&dev, bytes) != cudaSuccess) { free(host); return DLE_ERR_CUDA; }
    if (cudaMemcpy(dev, host, bytes, cudaMemcpyHostToDevice) != cudaSuccess) { cudaFree(dev); free(host); return DLE_ERR_CUDA; }
    free(host);
    LambPlan* pl = new LambPlan;
    uint8_t* d = static_cast<uint8_t*>(dev);
    pl->tensors = reinterpret_cast<LambTensorDev*>(d + o_t); pl->groups = reinterpret_cast<LambGroupDev*>(d + o_g);
    pl->chunks = reinterpret_cast<int2*>(d + o_c); pl->state = reinterpret_cast<LambState*>(d + o_s);
    pl->psq = reinterpret_cast<double*>(d + o_p); pl->usq = reinterpret_cast<double*>(d + o_u);
    pl->block = dev; pl->block_bytes = bytes; pl->n_tensors = n_tensors; pl->n_groups = n_groups;
    pl->n_chunks = (int)n_chunks; pl->grad_dtype = grad_dtype; pl->total_numel = total;
    pl->stage_numel = new long long[n_tensors];
    for (int i = 0; i < n_tensors; ++i) pl->stage_numel[i] = ht[i].numel;
    void* hs = nullptr;
    if (cudaMallocHost(&hs, sizeof(LambTensorDev) * (size_t)n_tensors * (LAMB_EAGER_SLOTS + LAMB_CAPTURE_SLOTS)) != cudaSuccess) {
        cudaFree(dev); delete[] pl->stage_numel; delete pl; return DLE_ERR_CUDA;
    }
    pl->host_stage = static_cast<LambTensorDev*>(hs);
    for (int i = 0; i < LAMB_EAGER_SLOTS; ++i)
        if (cudaEventCreateWithFlags(&pl->stage_event[i], cudaEventDisableTiming) != cudaSuccess) return DLE_ERR_CUDA;
    *plan_out = pl;
    return DLE_OK;
}

// Re-point an existing plan at new gradient / parameter addresses (same tensor count, sizes and groups): one small
// H2D copy on `stream`, no allocation, no host synchronisation, legal under CUDA-graph capture.  Autograd hands out fresh gradient tensors every step when the driver uses
// zero_grad(set_to_none=True) (run_pretraining.py:536), so this is on the per-step path.
extern "C" int dle_lamb_plan_update(void* plan, const dle_lamb_tensor* ht, int32_t n_tensors, void* stream) {
    DLE_CHECK_ARG(plan && ht);
    LambPlan* pl = static_cast<LambPlan*>(plan);
    DLE_CHECK_ARG(n_tensors == pl->n_tensors);
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
    if (cudaStreamIsCapturing(s, &cap) != cudaSuccess) return DLE_ERR_CUDA;
    int slot;
    if (cap == cudaStreamCaptureStatusActive) {
        if (pl->next_capture_slot >= LAMB_CAPTURE_SLOTS) return DLE_ERR_NOSYS;      // more graph captures than reserved slots
        slot = LAMB_EAGER_SLOTS + pl->next_capture_slot++;
    } else {
        slot = pl->next_slot;
        pl->next_slot = (pl->next_slot + 1) % LAMB_EAGER_SLOTS;
        // the slot was last read by the copy issued LAMB_EAGER_SLOTS updates ago: only a host running that far ahead ever waits here
        if (pl->stage_used[slot] && cudaEventQuery(pl->stage_event[slot]) == cudaErrorNotReady &&
            cudaEventSynchronize(pl->stage_event[slot]) != cudaSuccess) return DLE_ERR_CUDA;
    }
    LambTensorDev* t = pl->host_stage + (size_t)slot * n_tensors;
    for (int i = 0; i < n_tensors; ++i) {
        DLE_CHECK_ARG(ht[i].numel == pl->stage_numel[i] && ht[i].grad && ht[i].param && ht[i].exp_avg && ht[i].exp_avg_sq);
        t[i] = LambTensorDev{ht[i].grad, ht[i].param, ht[i].exp_avg, ht[i].exp_avg_sq, ht[i].model_param, ht[i].numel, ht[i].group, 0};
    }
    if (cudaMemcpyAsync(pl->tensors, t, sizeof(LambTensorDev) * n_tensors, cudaMemcpyHostToDevice, s) != cudaSuccess) return DLE_ERR_CUDA;
    if (cap != cudaStreamCaptureStatusActive) {
        if (cudaEventRecord(pl->stage_event[slot], s) != cudaSuccess) return DLE_ERR_CUDA;
        pl->stage_used[slot] = true;
    }
    return DLE_OK;
}

extern "C" int dle_lamb_plan_destroy(void* plan) {
    DLE_CHECK_ARG(plan);
    LambPlan* pl = static_cast<LambPlan*>(plan);
    cudaFree(pl->block);
    if (pl->host_stage) cudaFreeHost(pl->host_stage);
    for (int i = 0; i < LAMB_EAGER_SLOTS; ++i) if (pl->stage_event[i]) cudaEventDestroy(pl->stage_event[i]);
    delete[] pl->stage_numel;
    delete pl;
    return DLE_OK;
}

static int lamb_grad_pass_launch(LambPlan* pl, const float* scale, float max_grad_norm, float clip_eps, int advance, float* found_inf_out,
                                 float* gnorm_out, cudaStream_t s) {
    const int grid = lamb_grid(pl->n_chunks);
    if (pl->grad_dtype == DLE_DTYPE_BF16)
        lamb_grad_pass<bf16><<<grid, LAMB_THREADS, 0, s>>>(pl->tensors, pl->chunks, pl->n_chunks, pl->groups, pl->n_groups, pl->state,
                                                         pl->psq, pl->usq, pl->n_tensors, scale, max_grad_norm, clip_eps, advance, found_inf_out, gnorm_out);
    else
        lamb_grad_pass<float><<<grid, LAMB_THREADS, 0, s>>>(pl->tensors, pl->chunks, pl->n_chunks, pl->groups, pl->n_groups, pl->state,
                                                          pl->psq, pl->usq, pl->n_tensors, scale, max_grad_norm, clip_eps, advance, found_inf_out, gnorm_out);
    DLE_LAUNCH_CHECK();
    return DLE_OK;
}

extern "C" int dle_lamb_grad_norm(void* plan, float* norm_out, float* found_inf_out, void* stream) {
    DLE_CHECK_ARG(plan && norm_out);
    return lamb_grad_pass_launch(static_cast<LambPlan*>(plan), nullptr, 1.0f, 0.0f, 0, found_inf_out, norm_out,
                                 reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int dle_lamb_step(void* plan, const float* scale, float max_grad_norm, int32_t adam_w_mode, int32_t use_nvlamb,
                             float* found_inf_out, float* global_grad_norm_out, float* per_tensor_norms_out, void* stream) {
    DLE_CHECK_ARG(plan);
    LambPlan* pl = static_cast<LambPlan*>(plan);
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    int rc = lamb_grad_pass_launch(pl, scale, max_grad_norm, 0.0f, 1, found_inf_out, global_grad_norm_out, s);
    if (rc != DLE_OK) return rc;
    const int grid = lamb_grid(pl->n_chunks);
    if (pl->grad_dtype == DLE_DTYPE_BF16)
        lamb_stage1<bf16><<<grid, LAMB_THREADS, 0, s>>>(pl->tensors, pl->chunks, pl->n_chunks, pl->groups, pl->state, pl->psq, pl->usq, adam_w_mode);
    else
        lamb_stage1<float><<<grid, LAMB_THREADS, 0, s>>>(pl->tensors, pl->chunks, pl->n_chunks, pl->groups, pl->state, pl->psq, pl->usq, adam_w_mode);
    DLE_LAUNCH_CHECK();
    lamb_stage2<<<grid, LAMB_THREADS, 0, s>>>(pl->tensors, pl->chunks, pl->n_chunks, pl->groups, pl->state, pl->psq, pl->usq,
                                              adam_w_mode, use_nvlamb, per_tensor_norms_out, pl->n_tensors);
    DLE_LAUNCH_CHECK();
    return DLE_OK;
}

extern "C" int dle_adam_step(void* plan, const float* scale, float max_grad_norm, float clip_eps, int32_t adam_w_mode,
                             float* found_inf_out, float* global_grad_norm_out, void* stream) {
    DLE_CHECK_ARG(plan);
    LambPlan* pl = static_cast<LambPlan*>(plan);
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    int rc = lamb_grad_pass_launch(pl, scale, max_grad_norm, clip_eps, 1, found_inf_out, global_grad_norm_out, s);
    if (rc != DLE_OK) return rc;
    const int grid = lamb_grid(pl->n_chunks);
    if (pl->grad_dtype == DLE_DTYPE_BF16)
        adam_apply<bf16><<<grid, LAMB_THREADS, 0, s>>>(pl->tensors, pl->chunks, pl->n_chunks, pl->groups, pl->state, adam_w_mode);
    else
        adam_apply<float><<<grid, LAMB_THREADS, 0, s>>>(pl->tensors, pl->chunks, pl->n_chunks, pl->groups, pl->state, adam_w_mode);
    DLE_LAUNCH_CHECK();
    return DLE_OK;
}
