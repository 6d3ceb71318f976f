// vtp_b200 — linear probing on frozen trunk features (tools/test_linear_probing_hf.py): the feature assembly read in
// place from the residual stream, the per-classifier softmax cross-entropy with its bf16x3 gradient operand, the fused
// SGD-momentum step with the refresh of the next forward's weight operand, and the top-1 counts.  The classifier GEMMs
// themselves are vtp_gemm_bf16 (gemm.cu).  No atomics except the integer top-1 counts: every launch is bit-reproducible.
#include <math.h>

#include "host.h"
#include "ptx.cuh"

namespace vtp {

// ------------------------------------------------------------------------------------------------ features
// Row statistics of the trunk's final norm with the lane partition and reduction order of norm_fwd_kernel
// (elementwise.cu), so that a normalised cls row equals vtp_norm_fwd's fp32 output.
template <int MAXV>
__device__ __forceinline__ void probe_row_stats(const float* __restrict__ xr, int D, int lane, int is_ln, float eps,
                                                float& mean, float& rstd) {
    float v[MAXV][4];
    float s = 0.f;
#pragma unroll
    for (int g = 0; g < MAXV; ++g) {
        const int c = (g * 32 + lane) * 4;
        if (c < D) {
            const float4 t = *reinterpret_cast<const float4*>(xr + c);
            v[g][0] = t.x, v[g][1] = t.y, v[g][2] = t.z, v[g][3] = t.w;
            s += is_ln ? (v[g][0] + v[g][1] + v[g][2] + v[g][3])
                       : (v[g][0] * v[g][0] + v[g][1] * v[g][1] + v[g][2] * v[g][2] + v[g][3] * v[g][3]);
        }
    }
    s = warp_sum(s);
    mean = 0.f;
    if (is_ln) {
        mean = s / D;
        float q = 0.f;
#pragma unroll
        for (int g = 0; g < MAXV; ++g) {
            const int c = (g * 32 + lane) * 4;
            if (c < D) {
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const float d = v[g][i] - mean;
                    q += d * d;
                }
            }
        }
        q = warp_sum(q);
        rstd = rsqrtf(q / D + eps);
    } else {
        rstd = rsqrtf(s / D + eps);
    }
}

__device__ __forceinline__ float probe_norm1(float v, float mean, float rstd, float w, float b, int is_ln) {
    if (is_ln) return (v - mean) * rstd * w + b;
    const float n = v * rstd;
    return n * w;
}

// One CTA per image.  Phase 1: one warp per row computes (mean, rstd) into shared memory (only the cls row when no patch
// mean is wanted).  Phase 2: one thread per column writes the normalised cls value and sums the normalised patch rows in
// ascending token order.
template <int MAXV>
__global__ void __launch_bounds__(256) probe_features_kernel(const float* __restrict__ x, int T, int D,
                                                             const float* __restrict__ w, const float* __restrict__ b,
                                                             float eps, float* __restrict__ X, long ldX, int cls_col,
                                                             int mean_col) {
    extern __shared__ float sm[];
    const int rows = mean_col >= 0 ? T : 1;
    float* s_rstd = sm;
    float* s_mean = sm + rows;
    const float* xb = x + (long)blockIdx.x * T * D;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
    const int is_ln = b != nullptr;
    for (int r = warp; r < rows; r += nw) {
        float mean, rstd;
        probe_row_stats<MAXV>(xb + (long)r * D, D, lane, is_ln, eps, mean, rstd);
        if (lane == 0) s_rstd[r] = rstd, s_mean[r] = mean;
    }
    __syncthreads();
    float* Xb = X + (long)blockIdx.x * ldX;
    for (int c = threadIdx.x; c < D; c += blockDim.x) {
        const float wc = w[c], bc = is_ln ? b[c] : 0.f;
        Xb[cls_col + c] = probe_norm1(xb[c], s_mean[0], s_rstd[0], wc, bc, is_ln);
        if (mean_col >= 0) {
            float acc = 0.f;
#pragma unroll 4
            for (int t = 1; t < T; ++t) acc += probe_norm1(xb[(long)t * D + c], s_mean[t], s_rstd[t], wc, bc, is_ln);
            Xb[mean_col + c] = acc / (float)(T - 1);
        }
    }
}

// ------------------------------------------------------------------------------------------------ cross-entropy
// One CTA per classifier.  Phase 1: one warp per row -> row max, 1/Σexp, the row's loss.  Phase 2: one thread per column
// recomputes dZ = (softmax - onehot)/B row by row (same expression, same bits), writes its bf16x3 rows and sums the bias
// gradient in ascending row order.
__global__ void __launch_bounds__(512) probe_ce_kernel(const float* __restrict__ Z, long ldz, int B, int C, int Cp,
                                                       const long long* __restrict__ labels, float* __restrict__ loss_acc,
                                                       __nv_bfloat16* __restrict__ dZ3, long ldd,
                                                       float* __restrict__ dbias) {
    extern __shared__ float sm[];
    float* s_max = sm;
    float* s_inv = sm + B;
    int* s_lab = reinterpret_cast<int*>(sm + 2 * B);
    float* s_loss = sm + 3 * B;
    const int g = blockIdx.x;
    const float* Zg = Z + (long)g * Cp;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
    float part = 0.f;
    for (int r = warp; r < B; r += nw) {
        const float* z = Zg + (long)r * ldz;
        float m = -INFINITY;
        for (int c = lane; c < C; c += 32) m = fmaxf(m, z[c]);
        m = warp_max(m);
        float s = 0.f;
        for (int c = lane; c < C; c += 32) s += expf(z[c] - m);
        s = warp_sum(s);
        if (lane == 0) {
            const long long y = labels[r];
            const bool ok = y >= 0 && y < C;
            s_max[r] = m;
            s_inv[r] = 1.f / s;
            s_lab[r] = ok ? (int)y : -1;
            part += ok ? (m + logf(s)) - z[ok ? y : 0] : NAN;
        }
    }
    if (lane == 0) s_loss[warp] = part;
    __syncthreads();
    if (threadIdx.x == 0) {
        float t = 0.f;
        for (int i = 0; i < nw; ++i) t += s_loss[i];
        loss_acc[g] += t / B;
    }
    const float invB = 1.f / B;
    for (int c = threadIdx.x; c < Cp; c += blockDim.x) {
        float db = 0.f;
        __nv_bfloat16* o = dZ3 + (long)g * Cp + c;
        for (int r = 0; r < B; ++r) {
            float d = 0.f;
            if (c < C) d = (expf(Zg[(long)r * ldz + c] - s_max[r]) * s_inv[r] - (c == s_lab[r] ? 1.f : 0.f)) * invB;
            db += d;
            const float hi = bf16_round(d);
            const __nv_bfloat16 h = __float2bfloat16_rn(hi), l = __float2bfloat16_rn(d - hi);
            o[(long)r * ldd] = h;
            o[(long)(B + r) * ldd] = h;
            o[(long)(2 * B + r) * ldd] = l;
        }
        dbias[(long)g * Cp + c] = db;
    }
}

// ------------------------------------------------------------------------------------------------ SGD-momentum
// torch.optim.SGD's multi-tensor update, operation for operation: buf = clone(g) on the first step, else
// buf = (buf * momentum) + g (two roundings, as _foreach_mul_ then _foreach_add_); p = fma(-lr, buf, p) (_foreach_add_
// with alpha = -lr).  Four parameters per thread, all of one classifier (rows_per_cls * row_len % 4 == 0).
__global__ void probe_sgd_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ buf, long n4,
                                 int row_len, long per_cls, int cls0, const float* __restrict__ lr_tab, int lr_ld,
                                 int n_steps, const float* __restrict__ hyper, float mom, float gscale,
                                 __nv_bfloat16* __restrict__ pb) {
    const int step = (int)hyper[0];
    const int it = min(max(step, 1), n_steps) - 1;
    const float* lr_row = lr_tab + (long)it * lr_ld + cls0;
    const bool first = step <= 1;
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n4; i += (long)gridDim.x * blockDim.x) {
        const long e = i * 4;
        const float nlr = -lr_row[e / per_cls];
        const float4 gi = reinterpret_cast<const float4*>(g)[i];
        const float4 pi = reinterpret_cast<float4*>(p)[i];
        const float ga[4] = {gi.x * gscale, gi.y * gscale, gi.z * gscale, gi.w * gscale};
        float pa[4] = {pi.x, pi.y, pi.z, pi.w};
        float ba[4];
        if (first) {
#pragma unroll
            for (int k = 0; k < 4; ++k) ba[k] = ga[k];
        } else {
            const float4 bi = reinterpret_cast<float4*>(buf)[i];
            const float bo[4] = {bi.x, bi.y, bi.z, bi.w};
#pragma unroll
            for (int k = 0; k < 4; ++k) ba[k] = __fadd_rn(__fmul_rn(bo[k], mom), ga[k]);
        }
#pragma unroll
        for (int k = 0; k < 4; ++k) pa[k] = __fmaf_rn(nlr, ba[k], pa[k]);
        reinterpret_cast<float4*>(buf)[i] = make_float4(ba[0], ba[1], ba[2], ba[3]);
        reinterpret_cast<float4*>(p)[i] = make_float4(pa[0], pa[1], pa[2], pa[3]);
        if (pb) {  // hi|lo|hi, exactly split3_kernel's B side
            float hi[4], lo[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) hi[k] = bf16_round(pa[k]), lo[k] = pa[k] - hi[k];
            uint2 th, tl;
            th.x = pack_bf16x2(hi[0], hi[1]), th.y = pack_bf16x2(hi[2], hi[3]);
            tl.x = pack_bf16x2(lo[0], lo[1]), tl.y = pack_bf16x2(lo[2], lo[3]);
            __nv_bfloat16* o = pb + (e / row_len) * 3 * row_len + e % row_len;
            *reinterpret_cast<uint2*>(o) = th;
            *reinterpret_cast<uint2*>(o + row_len) = tl;
            *reinterpret_cast<uint2*>(o + 2 * row_len) = th;
        }
    }
}

// ------------------------------------------------------------------------------------------------ top-1
// torch.argmax order: NaN above every number, then larger value, then lower index.
__device__ __forceinline__ bool probe_better(float v, int i, float best, int bi) {
    const bool vn = isnan(v), bn = isnan(best);
    if (vn != bn) return vn;
    if (!vn && v != best) return v > best;
    return i < bi;
}

__global__ void __launch_bounds__(256) probe_correct_kernel(const float* __restrict__ Z, long ldz, int B, int C, int Cp,
                                                            const long long* __restrict__ labels,
                                                            unsigned long long* __restrict__ counts) {
    const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (row >= B) return;
    const float* z = Z + (long)row * ldz + (long)blockIdx.y * Cp;
    float best = -INFINITY;
    int bi = 0x7fffffff;
    for (int c = lane; c < C; c += 32) {
        const float v = z[c];
        if (probe_better(v, c, best, bi)) best = v, bi = c;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, best, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (probe_better(ov, oi, best, bi)) best = ov, bi = oi;
    }
    if (lane == 0 && (long long)bi == labels[row]) atomicAdd(counts + blockIdx.y, 1ULL);
}

static inline int probe_grid(long total, int block) {
    long g = (total + block - 1) / block;
    long cap = (long)num_sms() * 16;
    return (int)(g < cap ? (g > 0 ? g : 1) : cap);
}

}  // namespace vtp

using namespace vtp;

extern "C" int vtp_probe_features(const float* x, int B, int T, int D, const float* w, const float* b, float eps, float* X,
                                  long ldX, int cls_col, int mean_col, vtp_stream_t st) {
    VTP_CHECK_ARG(x && w && X && B > 0 && T >= 1 && cls_col >= 0, "probe_features: bad args");
    VTP_CHECK_ARG(D % 4 == 0 && D <= 2048, "probe_features: D must be a multiple of 4 and <= 2048");
    VTP_CHECK_ARG(mean_col < 0 || T >= 2, "probe_features: the patch mean needs T >= 2");
    VTP_CHECK_ARG(cls_col + D <= ldX && mean_col + D <= ldX, "probe_features: columns outside X's rows");
    const int rows = mean_col >= 0 ? T : 1;
    const size_t smem = 2 * sizeof(float) * rows;
    VTP_CHECK_ARG(smem <= 48 * 1024, "probe_features: T = %d exceeds the %d rows of shared memory statistics", T,
                  48 * 1024 / 8);
    cudaStream_t s = (cudaStream_t)st;
#define LAUNCH_FEAT(MV) \
    probe_features_kernel<MV><<<B, 256, smem, s>>>(x, T, D, w, b, eps, X, ldX, cls_col, mean_col)
    if (D <= 512) LAUNCH_FEAT(4);
    else if (D <= 1024) LAUNCH_FEAT(8);
    else LAUNCH_FEAT(16);
#undef LAUNCH_FEAT
    VTP_LAUNCH_CHECK();
    return VTP_OK;
}

extern "C" int vtp_probe_ce(const float* Z, long ldz, int B, int G, int C, int Cp, const int64_t* labels, float* loss_acc,
                            void* dZ3, long ldd, float* dbias, vtp_stream_t st) {
    VTP_CHECK_ARG(Z && labels && loss_acc && dZ3 && dbias && B > 0 && G > 0 && C > 0, "probe_ce: bad args");
    VTP_CHECK_ARG(Cp >= C && ldz >= (long)G * Cp && ldd >= (long)G * Cp, "probe_ce: bad strides");
    const size_t smem = sizeof(float) * (3 * (size_t)B + 16);
    VTP_CHECK_ARG(smem <= 48 * 1024, "probe_ce: batch %d too large", B);
    probe_ce_kernel<<<G, 512, smem, (cudaStream_t)st>>>(Z, ldz, B, C, Cp, (const long long*)labels, loss_acc,
                                                         (__nv_bfloat16*)dZ3, ldd, dbias);
    VTP_LAUNCH_CHECK();
    return VTP_OK;
}

extern "C" int vtp_probe_sgd(float* p, const float* g, float* buf, long n, int row_len, int rows_per_cls, int cls0,
                             const float* lr_table, int lr_ld, int n_steps, const float* hyper, float momentum,
                             float gscale, void* pb, vtp_stream_t st) {
    VTP_CHECK_ARG(p && g && buf && lr_table && hyper && n > 0 && row_len > 0 && rows_per_cls > 0 && cls0 >= 0 &&
                      n_steps > 0 && lr_ld > 0,
                  "probe_sgd: bad args");
    const long per_cls = (long)rows_per_cls * row_len;
    VTP_CHECK_ARG(n % 4 == 0 && per_cls % 4 == 0 && (!pb || row_len % 4 == 0),
                  "probe_sgd: n, rows_per_cls * row_len (and row_len with pb) must be multiples of 4");
    VTP_CHECK_ARG(cls0 + (n - 1) / per_cls < lr_ld, "probe_sgd: classifier index past the lr table's row");
    probe_sgd_kernel<<<probe_grid(n / 4, 256), 256, 0, (cudaStream_t)st>>>(p, g, buf, n / 4, row_len, per_cls, cls0,
                                                                           lr_table, lr_ld, n_steps, hyper, momentum,
                                                                           gscale, (__nv_bfloat16*)pb);
    VTP_LAUNCH_CHECK();
    return VTP_OK;
}

extern "C" int vtp_probe_correct(const float* Z, long ldz, int B, int G, int C, int Cp, const int64_t* labels,
                                 int64_t* counts, vtp_stream_t st) {
    VTP_CHECK_ARG(Z && labels && counts && B > 0 && G > 0 && C > 0 && Cp >= C && ldz >= (long)G * Cp && G <= 65535,
                  "probe_correct: bad args");
    dim3 grid(ceil_div(B, 8), G);
    probe_correct_kernel<<<grid, 256, 0, (cudaStream_t)st>>>(Z, ldz, B, C, Cp, (const long long*)labels,
                                                             (unsigned long long*)counts);
    VTP_LAUNCH_CHECK();
    return VTP_OK;
}
