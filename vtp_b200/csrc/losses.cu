// vtp_b200 — loss heads of the 3-objective step, forward value + gradient in one pass over the logits.
// The reference ships NO loss code (SURVEY.md M3): these restate OpenCLIP ClipLoss (softmax cross-entropy over the
// gathered similarity matrix), DINOv2 DINOLoss / iBOTPatchLoss (centred+sharpened teacher softmax vs student
// log-softmax over K prototypes) and an L1 pixel loss; oracle/vtp_oracle.py holds the matching CPU definitions.
#include "host.h"
#include "ptx.cuh"

namespace vtp {

__device__ __forceinline__ float block_reduce(float v, float* sh, bool is_max) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
    v = is_max ? warp_max(v) : warp_sum(v);
    __syncthreads();
    if (lane == 0) sh[warp] = v;
    __syncthreads();
    float r = (threadIdx.x < nw) ? sh[threadIdx.x] : (is_max ? -INFINITY : 0.f);
    if (warp == 0) {
        r = is_max ? warp_max(r) : warp_sum(r);
        if (lane == 0) sh[0] = r;
    }
    __syncthreads();
    return sh[0];
}

// ------------------------------------------------------------------------------------------------ contrastive CE
// sim fp32 [R][ld] (C valid columns) = I·Tᵀ block; logits = exp(*log_scale) * sim (log_scale may be NULL -> 1);
// label(r) = label0 + r.
//   loss_acc   += coef * Σ_r (lse_r − logit[r,label])
//   dscale_acc += Σ_r Σ_c g[r,c] * logit[r,c]           (= d loss / d log_scale),  g = coef (softmax − onehot)
//   G bf16 [R][ldg] = exp(log_scale) * g                   (= d loss / d sim, the operand of the feature-grad GEMMs)
__global__ void softmax_ce_kernel(const float* __restrict__ logits, long ld, int C, int label0,
                                  const float* __restrict__ log_scale, __nv_bfloat16* __restrict__ G, long ldg, float coef,
                                  float* __restrict__ loss_acc, float* __restrict__ dscale_acc) {
    __shared__ float sh[32];
    const int r = blockIdx.x;
    const float sc = log_scale ? __expf(*log_scale) : 1.f;
    const float* lr = logits + (long)r * ld;
    float m = -INFINITY;
    for (int c = threadIdx.x; c < C; c += blockDim.x) m = fmaxf(m, sc * lr[c]);
    m = block_reduce(m, sh, true);
    float s = 0.f;
    for (int c = threadIdx.x; c < C; c += blockDim.x) s += __expf(sc * lr[c] - m);
    s = block_reduce(s, sh, false);
    const float lse = m + logf(s);
    const int label = label0 + r;
    float ds = 0.f;
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
        const float x = sc * lr[c];
        const float g = coef * (__expf(x - lse) - (c == label ? 1.f : 0.f));
        ds += g * x;
        G[(long)r * ldg + c] = __float2bfloat16_rn(sc * g);
    }
    ds = block_reduce(ds, sh, false);
    if (threadIdx.x == 0) {
        atomicAdd(loss_acc, coef * (lse - sc * lr[label]));
        if (dscale_acc) atomicAdd(dscale_acc, ds);
    }
}

// ------------------------------------------------------------------------------------------------ DINO / iBOT
// teacher: probs[r,:] = softmax((t[r,:] − center) / temp), in place (bf16).  One block per row; the row is read from
// HBM once (16-byte vector loads), cached in shared memory as raw bf16, and written once.  K % 8 == 0.
__device__ __forceinline__ void unpack8(const uint4& q, float (&f)[8]) {
    f[0] = bf16_lo(q.x), f[1] = bf16_hi(q.x), f[2] = bf16_lo(q.y), f[3] = bf16_hi(q.y);
    f[4] = bf16_lo(q.z), f[5] = bf16_hi(q.z), f[6] = bf16_lo(q.w), f[7] = bf16_hi(q.w);
}
__device__ __forceinline__ uint4 pack8(const float (&f)[8]) {
    uint4 q;
    q.x = pack_bf16x2(f[0], f[1]), q.y = pack_bf16x2(f[2], f[3]), q.z = pack_bf16x2(f[4], f[5]), q.w = pack_bf16x2(f[6], f[7]);
    return q;
}

// Instruction- and occupancy-lean form: 1024 threads per
// row block (32 warps/SM), base-2 exponentials with the temperature folded into one FFMA per element, every pass fully
// vectorised on 16-byte shared / global accesses.
__device__ __forceinline__ float ex2_approx(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

__global__ void __launch_bounds__(1024, 1)
dino_teacher_kernel(__nv_bfloat16* __restrict__ t, const float* __restrict__ center, int K, float inv_temp) {
    extern __shared__ uint4 rowq[];  // K/8 packed bf16x8 (128 KB at K = 65536)
    __shared__ float sh[32];
    uint4* tr = reinterpret_cast<uint4*>(t + (long)blockIdx.x * K);
    const float4* c4 = reinterpret_cast<const float4*>(center);
    const int K8 = K >> 3;
    const float it2 = inv_temp * 1.4426950408889634f;   // exp(z / temp) = 2^(z * it2)
    float m = -INFINITY;                                // max of (t - c): inv_temp > 0, scale once afterwards
    for (int c = threadIdx.x; c < K8; c += blockDim.x) {
        const uint4 q = tr[c];
        rowq[c] = q;
        float f[8];
        unpack8(q, f);
        const float4 a = __ldg(c4 + 2 * c), b = __ldg(c4 + 2 * c + 1);
        m = fmaxf(m, fmaxf(fmaxf(f[0] - a.x, f[1] - a.y), fmaxf(f[2] - a.z, f[3] - a.w)));
        m = fmaxf(m, fmaxf(fmaxf(f[4] - b.x, f[5] - b.y), fmaxf(f[6] - b.z, f[7] - b.w)));
    }
    m = block_reduce(m, sh, true);
    const float m2 = m * it2;
    float s0 = 0.f, s1 = 0.f;
    for (int c = threadIdx.x; c < K8; c += blockDim.x) {
        float f[8];
        unpack8(rowq[c], f);
        const float4 a = __ldg(c4 + 2 * c), b = __ldg(c4 + 2 * c + 1);
        s0 += ex2_approx(fmaf(f[0] - a.x, it2, -m2)) + ex2_approx(fmaf(f[1] - a.y, it2, -m2)) +
              ex2_approx(fmaf(f[2] - a.z, it2, -m2)) + ex2_approx(fmaf(f[3] - a.w, it2, -m2));
        s1 += ex2_approx(fmaf(f[4] - b.x, it2, -m2)) + ex2_approx(fmaf(f[5] - b.y, it2, -m2)) +
              ex2_approx(fmaf(f[6] - b.z, it2, -m2)) + ex2_approx(fmaf(f[7] - b.w, it2, -m2));
    }
    const float ssum = block_reduce(s0 + s1, sh, false);
    const float l2 = m2 + log2f(ssum);                  // log2 of the partition function
    for (int c = threadIdx.x; c < K8; c += blockDim.x) {
        float f[8];
        unpack8(rowq[c], f);
        const float4 a = __ldg(c4 + 2 * c), b = __ldg(c4 + 2 * c + 1);
        f[0] = ex2_approx(fmaf(f[0] - a.x, it2, -l2)), f[1] = ex2_approx(fmaf(f[1] - a.y, it2, -l2));
        f[2] = ex2_approx(fmaf(f[2] - a.z, it2, -l2)), f[3] = ex2_approx(fmaf(f[3] - a.w, it2, -l2));
        f[4] = ex2_approx(fmaf(f[4] - b.x, it2, -l2)), f[5] = ex2_approx(fmaf(f[5] - b.y, it2, -l2));
        f[6] = ex2_approx(fmaf(f[6] - b.z, it2, -l2)), f[7] = ex2_approx(fmaf(f[7] - b.w, it2, -l2));
        tr[c] = pack8(f);
    }
}

// student: for row r with teacher rows t0[r], t1[r] (−1 = none; either may be −1, t1 may be NULL), weight w[r]:
//   z = s/τ ;  loss += w Σ_v (lse(z) − Σ_k T_v[k] z[k]) ;  ds[k] = (w/τ) (n_v softmax(z)[k] − Σ_v T_v[k])   (in place, bf16)
// A row without teachers gets zero loss and gradient.
__global__ void __launch_bounds__(1024, 1)
dino_student_kernel(__nv_bfloat16* __restrict__ s, const __nv_bfloat16* __restrict__ tprobs,
                    const int* __restrict__ t0, const int* __restrict__ t1, const float* __restrict__ w,
                    int K, float inv_temp, float* __restrict__ loss_acc) {
    extern __shared__ uint4 rowq[];  // K/8 packed student logits
    __shared__ float sh[32];
    const int r = blockIdx.x;
    uint4* sr = reinterpret_cast<uint4*>(s + (long)r * K);
    const int i0 = t0[r], i1 = t1 ? t1[r] : -1;
    const float wr = w[r];
    const uint4* ta = i0 >= 0 ? reinterpret_cast<const uint4*>(tprobs + (long)i0 * K) : nullptr;
    const uint4* tb = i1 >= 0 ? reinterpret_cast<const uint4*>(tprobs + (long)i1 * K) : nullptr;
    if (!ta) ta = tb, tb = nullptr;   // the teacher terms below are read under `if (ta)`: a lone t1 moves to the first slot
    const float nv = (ta ? 1.f : 0.f) + (tb ? 1.f : 0.f);
    const int K8 = K >> 3;
    const float it2 = inv_temp * 1.4426950408889634f;
    float m = -INFINITY, dot = 0.f;                     // max of the raw logits; dot = Σ_k T[k] s[k] (scaled afterwards)
    for (int c = threadIdx.x; c < K8; c += blockDim.x) {
        const uint4 q = sr[c];
        rowq[c] = q;
        float z[8], tt[8];
        unpack8(q, z);
        m = fmaxf(m, fmaxf(fmaxf(fmaxf(z[0], z[1]), fmaxf(z[2], z[3])), fmaxf(fmaxf(z[4], z[5]), fmaxf(z[6], z[7]))));
        if (ta) {
            unpack8(__ldg(ta + c), tt);
            if (tb) {
                float f[8];
                unpack8(__ldg(tb + c), f);
#pragma unroll
                for (int i = 0; i < 8; ++i) tt[i] += f[i];
            }
#pragma unroll
            for (int i = 0; i < 8; ++i) dot = fmaf(tt[i], z[i], dot);
        }
    }
    m = block_reduce(m, sh, true);
    dot = block_reduce(dot, sh, false) * inv_temp;
    const float m2 = m * it2;
    float se0 = 0.f, se1 = 0.f;
    for (int c = threadIdx.x; c < K8; c += blockDim.x) {
        float z[8];
        unpack8(rowq[c], z);
        se0 += ex2_approx(fmaf(z[0], it2, -m2)) + ex2_approx(fmaf(z[1], it2, -m2)) + ex2_approx(fmaf(z[2], it2, -m2)) +
               ex2_approx(fmaf(z[3], it2, -m2));
        se1 += ex2_approx(fmaf(z[4], it2, -m2)) + ex2_approx(fmaf(z[5], it2, -m2)) + ex2_approx(fmaf(z[6], it2, -m2)) +
               ex2_approx(fmaf(z[7], it2, -m2));
    }
    const float se = block_reduce(se0 + se1, sh, false);
    const float l2 = m2 + log2f(se);
    const float lse = l2 * 0.6931471805599453f;         // natural-log partition function of z = s / temp
    const float gscale = wr * inv_temp, gn = gscale * nv;
    for (int c = threadIdx.x; c < K8; c += blockDim.x) {
        float z[8], tt[8];
        unpack8(rowq[c], z);
#pragma unroll
        for (int i = 0; i < 8; ++i) tt[i] = 0.f;
        if (ta) {
            unpack8(__ldg(ta + c), tt);
            if (tb) {
                float f[8];
                unpack8(__ldg(tb + c), f);
#pragma unroll
                for (int i = 0; i < 8; ++i) tt[i] += f[i];
            }
        }
#pragma unroll
        for (int i = 0; i < 8; ++i) z[i] = fmaf(gn, ex2_approx(fmaf(z[i], it2, -l2)), -gscale * tt[i]);
        sr[c] = pack8(z);
    }
    if (threadIdx.x == 0) atomicAdd(loss_acc, wr * (nv * lse - dot));
}

// ------------------------------------------------------------------------------------------------ reconstruction L1
// rec (bf16|fp32) NCHW [B,C,H,W], tgt fp32 NCHW ; dlp optional fp32 NCHW extra gradient (LPIPS) ;
//   loss_acc += coef * Σ|rec − tgt|     out bf16 [B*gh*gw][C*r*r] = coef*sign(rec − tgt) + dlp   (pixel-unshuffled:
//   the dY operand of proj_out's dgrad/wgrad, decoders/pixel_decoder.py:157-160)
template <typename TR>
__global__ void recon_grad_kernel(const TR* __restrict__ rec, const float* __restrict__ tgt, const float* __restrict__ dlp,
                                  __nv_bfloat16* __restrict__ out, float* __restrict__ loss_acc, int B, int C, int gh,
                                  int gw, int r, float coef) {
    __shared__ float sh[32];
    const int N = C * r * r;
    const long total = (long)B * gh * gw * N;
    const int H = gh * r, W = gw * r;
    float acc = 0.f;
    for (long t = blockIdx.x * (long)blockDim.x + threadIdx.x; t < total; t += (long)gridDim.x * blockDim.x) {
        const int col = (int)(t % N);
        const long row = t / N;
        const int c = col / (r * r), ii = (col / r) % r, jj = col % r;
        const int b = (int)(row / (gh * gw)), hi = (int)((row / gw) % gh), wi = (int)(row % gw);
        const long idx = (((long)b * C + c) * H + hi * r + ii) * W + wi * r + jj;
        const float d = (float)rec[idx] - tgt[idx];
        acc += fabsf(d);
        float g = coef * (d > 0.f ? 1.f : (d < 0.f ? -1.f : 0.f));
        if (dlp) g += dlp[idx];
        out[t] = __float2bfloat16_rn(g);
    }
    acc = block_reduce(acc, sh, false);
    if (threadIdx.x == 0) atomicAdd(loss_acc, coef * acc);
}

// y = a*y + b*x  (teacher-centre EMA, misc)
__global__ void axpby_kernel(float* __restrict__ y, const float* __restrict__ x, float a, float b, long n) {
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x)
        y[i] = a * y[i] + b * x[i];
}

}  // namespace vtp

using namespace vtp;

extern "C" int vtp_softmax_ce(const float* logits, long ld, int R, int C, int label0, const float* log_scale, void* G_bf16,
                              long ldg, float coef, float* loss_acc, float* dscale_acc, vtp_stream_t st) {
    VTP_CHECK_ARG(logits && G_bf16 && loss_acc && R > 0 && C > 0 && label0 >= 0 && label0 + R <= C, "softmax_ce: bad args");
    softmax_ce_kernel<<<R, 256, 0, (cudaStream_t)st>>>(logits, ld, C, label0, log_scale, (__nv_bfloat16*)G_bf16, ldg, coef,
                                                       loss_acc, dscale_acc);
    VTP_LAUNCH_CHECK();
    return VTP_OK;
}

extern "C" int vtp_dino_teacher_probs(void* t_bf16, const float* center, int R, int K, float temp, vtp_stream_t st) {
    VTP_CHECK_ARG(t_bf16 && center && R > 0 && K > 0 && K % 8 == 0 && temp > 0, "dino_teacher_probs: bad args (K %% 8 == 0)");
    const size_t smem = (size_t)K * sizeof(__nv_bfloat16);
    VTP_CHECK_ARG(smem <= 220 * 1024, "dino_teacher_probs: K=%d too large for the smem-resident row", K);
    static size_t conf = 0;
    if (smem > conf) {
        VTP_CUDA(cudaFuncSetAttribute(dino_teacher_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        conf = smem;
    }
    dino_teacher_kernel<<<R, 1024, smem, (cudaStream_t)st>>>((__nv_bfloat16*)t_bf16, center, K, 1.f / temp);
    VTP_LAUNCH_CHECK();
    return VTP_OK;
}

extern "C" int vtp_dino_student_ce(void* s_bf16, const void* tprobs_bf16, const int* t0, const int* t1, const float* w,
                                   int R, int K, float temp, float* loss_acc, vtp_stream_t st) {
    VTP_CHECK_ARG(s_bf16 && tprobs_bf16 && t0 && w && loss_acc && R > 0 && K > 0 && K % 8 == 0 && temp > 0,
                  "dino_student_ce: bad args (K %% 8 == 0)");
    const size_t smem = (size_t)K * sizeof(__nv_bfloat16);
    VTP_CHECK_ARG(smem <= 220 * 1024, "dino_student_ce: K=%d too large for the smem-resident row", K);
    static size_t conf = 0;
    if (smem > conf) {
        VTP_CUDA(cudaFuncSetAttribute(dino_student_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        conf = smem;
    }
    dino_student_kernel<<<R, 1024, smem, (cudaStream_t)st>>>((__nv_bfloat16*)s_bf16, (const __nv_bfloat16*)tprobs_bf16, t0, t1,
                                                          w, K, 1.f / temp, loss_acc);
    VTP_LAUNCH_CHECK();
    return VTP_OK;
}

extern "C" int vtp_recon_l1_grad(const void* rec, int rec_dtype, const float* tgt, const float* dlp, void* out_bf16,
                                 float* loss_acc, int B, int C, int gh, int gw, int r, float coef, vtp_stream_t st) {
    VTP_CHECK_ARG(rec && tgt && out_bf16 && loss_acc && B > 0, "recon_l1_grad: bad args");
    const long total = (long)B * gh * gw * C * r * r;
    long g = (total + 255) / 256;
    const int grid = (int)(g < (long)num_sms() * 8 ? g : (long)num_sms() * 8);
    if (rec_dtype == VTP_F32)
        recon_grad_kernel<float><<<grid, 256, 0, (cudaStream_t)st>>>((const float*)rec, tgt, dlp, (__nv_bfloat16*)out_bf16,
                                                                    loss_acc, B, C, gh, gw, r, coef);
    else
        recon_grad_kernel<__nv_bfloat16><<<grid, 256, 0, (cudaStream_t)st>>>(
            (const __nv_bfloat16*)rec, tgt, dlp, (__nv_bfloat16*)out_bf16, loss_acc, B, C, gh, gw, r, coef);
    VTP_LAUNCH_CHECK();
    return VTP_OK;
}

extern "C" int vtp_axpby(float* y, const float* x, float a, float b, long n, vtp_stream_t st) {
    VTP_CHECK_ARG(y && x && n > 0, "axpby: bad args");
    long g = (n + 255) / 256;
    axpby_kernel<<<(int)(g < 4096 ? g : 4096), 256, 0, (cudaStream_t)st>>>(y, x, a, b, n);
    VTP_LAUNCH_CHECK();
    return VTP_OK;
}
