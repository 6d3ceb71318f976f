// vtp_b200 — zero-shot classification (tools/test_zero_shot_hf.py): the prompt-ensemble classifier from per-prompt text
// features, the image-side operand of the logits GEMM, and the target-rank count behind top-k accuracy.  The logits
// themselves are vtp_gemm_bf16 (gemm.cu).  No atomics except the integer hit counters: every output is bit-reproducible.
#include <math.h>

#include "host.h"
#include "ptx.cuh"

namespace vtp {

__device__ __forceinline__ float zs_load(const void* p, int dtype, long i) {
    return dtype == VTP_BF16 ? __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(p)[i])
                             : reinterpret_cast<const float*>(p)[i];
}

// Sum of a per-thread partial over the CTA (fixed order: warp shuffles, then warps in ascending order).
__device__ __forceinline__ float zs_block_sum(float v, float* s_red) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
    v = warp_sum(v);
    __syncthreads();  // s_red may still be read by a previous call
    if (lane == 0) s_red[warp] = v;
    __syncthreads();
    float t = 0.f;
    for (int i = 0; i < nw; ++i) t += s_red[i];
    return t;
}

// ------------------------------------------------------------------------------------------------ class embeddings
// One CTA per (padded) class.  Phase 1: one warp per template row -> the row's fp32 L2 norm clamped at eps (shared
// memory).  Phase 2: each thread owns columns c = tid + k*blockDim and sums x / denom over the templates in ascending
// order, divides by T (the template mean), then the mean row is normalised the same way.
template <int MAXC>
__global__ void __launch_bounds__(256) zs_class_embed_kernel(const void* __restrict__ feat, int dtype,
                                                             const int* __restrict__ row_of, int C, int T, int E,
                                                             float* __restrict__ out) {
    extern __shared__ float sm[];
    float* s_den = sm;        // [T]
    float* s_red = sm + T;    // [8]
    const int cls = blockIdx.x;
    float* o = out + (long)cls * E;
    if (cls >= C) {
        for (int c = threadIdx.x; c < E; c += blockDim.x) o[c] = 0.f;
        return;
    }
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
    for (int t = warp; t < T; t += nw) {
        const long p = (long)cls * T + t;
        const long r = row_of ? (long)row_of[p] : p;
        float s = 0.f;
        for (int c = lane; c < E; c += 32) {
            const float v = zs_load(feat, dtype, r * E + c);
            s = __fmaf_rn(v, v, s);
        }
        s = warp_sum(s);
        if (lane == 0) s_den[t] = fmaxf(sqrtf(s), 1e-12f);
    }
    __syncthreads();
    float acc[MAXC];
#pragma unroll
    for (int k = 0; k < MAXC; ++k) acc[k] = 0.f;
    for (int t = 0; t < T; ++t) {
        const long p = (long)cls * T + t;
        const long r = row_of ? (long)row_of[p] : p;
        const float d = s_den[t];
#pragma unroll
        for (int k = 0; k < MAXC; ++k) {
            const int c = threadIdx.x + k * blockDim.x;
            if (c < E) acc[k] += __fdiv_rn(zs_load(feat, dtype, r * E + c), d);
        }
    }
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < MAXC; ++k) {
        acc[k] = __fdiv_rn(acc[k], (float)T);
        if (threadIdx.x + k * blockDim.x < E) s = __fmaf_rn(acc[k], acc[k], s);
    }
    const float d = fmaxf(sqrtf(zs_block_sum(s, s_red)), 1e-12f);
#pragma unroll
    for (int k = 0; k < MAXC; ++k) {
        const int c = threadIdx.x + k * blockDim.x;
        if (c < E) o[c] = __fdiv_rn(acc[k], d);
    }
}

// ------------------------------------------------------------------------------------------------ image operand
// One warp per row: a = fl32(scale * fl32(x / max(||x||, eps))), written as fp32 or rounded once to bf16.
__global__ void __launch_bounds__(256) zs_image_operand_kernel(const void* __restrict__ x, int x_dtype, int B, int E,
                                                               float scale, void* __restrict__ out, int out_dtype) {
    const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (row >= B) return;
    const long base = (long)row * E;
    float s = 0.f;
    for (int c = lane; c < E; c += 32) {
        const float v = zs_load(x, x_dtype, base + c);
        s = __fmaf_rn(v, v, s);
    }
    const float d = fmaxf(sqrtf(warp_sum(s)), 1e-12f);
    for (int c = lane; c < E; c += 32) {
        const float a = __fmul_rn(scale, __fdiv_rn(zs_load(x, x_dtype, base + c), d));
        if (out_dtype == VTP_BF16) reinterpret_cast<__nv_bfloat16*>(out)[base + c] = __float2bfloat16_rn(a);
        else reinterpret_cast<float*>(out)[base + c] = a;
    }
}

// ------------------------------------------------------------------------------------------------ target rank
// torch.sort / torch.topk order: NaN above every number, then larger value; ties go to the lower index.
__device__ __forceinline__ bool zs_ahead(float v, int j, float lt, int t) {
    const bool vn = isnan(v), tn = isnan(lt);
    if (vn != tn) return vn;
    if (!vn && v != lt) return v > lt;
    return j < t;
}

struct ZsKs {
    int n;
    int k[VTP_ZS_MAX_K];
};

// One warp per row: rank = #{j : logit j is ahead of the target's}; rank C for a target outside [0, C).  Hits are
// counted per CTA in shared memory, then added to the int64 counters with one atomic per k.
__global__ void __launch_bounds__(256) zs_rank_kernel(const void* __restrict__ logits, int dtype, long ld, int B, int C,
                                                      const long long* __restrict__ targets, ZsKs ks,
                                                      int* __restrict__ ranks, unsigned long long* __restrict__ counts) {
    __shared__ unsigned int s_hits[VTP_ZS_MAX_K];
    if (threadIdx.x < VTP_ZS_MAX_K) s_hits[threadIdx.x] = 0u;
    __syncthreads();
    const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (row < B) {
        const long long tg = targets[row];
        int rank = C;
        if (tg >= 0 && tg < C) {
            const int t = (int)tg;
            const long base = (long)row * ld;
            const float lt = zs_load(logits, dtype, base + t);
            int n = 0;
            for (int j = lane; j < C; j += 32) n += zs_ahead(zs_load(logits, dtype, base + j), j, lt, t) ? 1 : 0;
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) n += __shfl_xor_sync(0xffffffffu, n, o);
            rank = n;
        }
        if (lane == 0) {
            ranks[row] = rank;
            for (int i = 0; i < ks.n; ++i)
                if (rank < ks.k[i]) atomicAdd(&s_hits[i], 1u);
        }
    }
    __syncthreads();
    if (threadIdx.x < ks.n && s_hits[threadIdx.x]) atomicAdd(counts + threadIdx.x, (unsigned long long)s_hits[threadIdx.x]);
}

}  // namespace vtp

using namespace vtp;

extern "C" int vtp_zs_class_embed(const void* feat, int feat_dtype, const int* row_of, int C, int T, int E, int Cp,
                                  float* out, vtp_stream_t st) {
    VTP_CHECK_ARG(feat && out && C > 0 && T > 0 && E > 0 && Cp >= C, "zs_class_embed: bad args");
    VTP_CHECK_ARG(feat_dtype == VTP_F32 || feat_dtype == VTP_BF16, "zs_class_embed: features must be fp32 or bf16");
    VTP_CHECK_ARG(E <= 1024, "zs_class_embed: E = %d exceeds 1024", E);
    const size_t smem = sizeof(float) * ((size_t)T + 8);
    VTP_CHECK_ARG(smem <= 48 * 1024, "zs_class_embed: T = %d templates exceed shared memory", T);
    cudaStream_t s = (cudaStream_t)st;
#define LAUNCH_CE(MC) zs_class_embed_kernel<MC><<<Cp, 256, smem, s>>>(feat, feat_dtype, row_of, C, T, E, out)
    if (E <= 512) LAUNCH_CE(2);
    else LAUNCH_CE(4);
#undef LAUNCH_CE
    VTP_LAUNCH_CHECK();
    return VTP_OK;
}

extern "C" int vtp_zs_image_operand(const void* x, int x_dtype, int B, int E, float scale, void* out, int out_dtype,
                                    vtp_stream_t st) {
    VTP_CHECK_ARG(x && out && B > 0 && E > 0, "zs_image_operand: bad args");
    VTP_CHECK_ARG((x_dtype == VTP_F32 || x_dtype == VTP_BF16) && (out_dtype == VTP_F32 || out_dtype == VTP_BF16),
                  "zs_image_operand: dtypes must be fp32 or bf16");
    zs_image_operand_kernel<<<ceil_div(B, 8), 256, 0, (cudaStream_t)st>>>(x, x_dtype, B, E, scale, out, out_dtype);
    VTP_LAUNCH_CHECK();
    return VTP_OK;
}

extern "C" int vtp_zs_rank(const void* logits, int dtype, long ld, int B, int C, const int64_t* targets, const int* ks,
                           int nk, int* ranks, int64_t* counts, vtp_stream_t st) {
    VTP_CHECK_ARG(logits && targets && ranks && B > 0 && C > 0 && ld >= C, "zs_rank: bad args");
    VTP_CHECK_ARG(dtype == VTP_F32 || dtype == VTP_BF16, "zs_rank: logits must be fp32 or bf16");
    VTP_CHECK_ARG(nk >= 0 && nk <= VTP_ZS_MAX_K && (nk == 0 || (ks && counts)), "zs_rank: 0..%d values of k",
                  VTP_ZS_MAX_K);
    ZsKs kk;
    kk.n = nk;
    for (int i = 0; i < VTP_ZS_MAX_K; ++i) kk.k[i] = i < nk ? ks[i] : 0;
    zs_rank_kernel<<<ceil_div(B, 8), 256, 0, (cudaStream_t)st>>>(logits, dtype, ld, B, C, (const long long*)targets, kk,
                                                                 ranks, (unsigned long long*)counts);
    VTP_LAUNCH_CHECK();
    return VTP_OK;
}
