// vtp_b200 — HBM-bound forward kernels around the GEMMs: im2col (patchify), token assembly, RMSNorm/LayerNorm,
// layout transposes, bf16x3 operand splitting.  All are single-pass, 16-byte vectorised, one warp per row where a
// row reduction is needed (D <= 2048 stays in registers).
#include "host.h"
#include "ptx.cuh"

namespace vtp {

// ------------------------------------------------------------------------------------------------ patchify
// img fp32 [B,C,H,W] -> out bf16 [B*gh*gw][C*p*p], k = c*p*p + i*p + j  (== Conv2d weight.flatten(1) order,
// layers/embeddings.py:58).  One thread handles 4 consecutive j (16B load, 8B store).
template <typename TO>
__global__ void patchify_kernel(const float* __restrict__ img, TO* __restrict__ out, int B, int C, int H,
                                int W, int p, long total4) {
    const int gw = W / p, gh = H / p, K = C * p * p;
    for (long t = blockIdx.x * (long)blockDim.x + threadIdx.x; t < total4; t += (long)gridDim.x * blockDim.x) {
        const long e = t * 4;  // flat index into out
        const long row = e / K;
        const int k = (int)(e % K);
        const int c = k / (p * p), i = (k / p) % p, j = k % p;
        const int b = (int)(row / (gh * gw)), ph = (int)((row / gw) % gh), pw = (int)(row % gw);
        const float4 v =
            __ldg(reinterpret_cast<const float4*>(img + (((long)b * C + c) * H + ph * p + i) * W + pw * p + j));
        if constexpr (sizeof(TO) == 4) {
            *reinterpret_cast<float4*>(out + e) = v;
        } else {
            uint2 w;
            w.x = pack_bf16x2(v.x, v.y), w.y = pack_bf16x2(v.z, v.w);
            *reinterpret_cast<uint2*>(out + e) = w;
        }
    }
}

// ------------------------------------------------------------------------------------------------ token rows
// x[(b*T + t) * D + :] = vec[t*D + :]  for t < nprefix  (cls / storage tokens); x fp32 or bf16
template <typename T>
__global__ void fill_prefix_kernel(T* __restrict__ x, const float* __restrict__ vec, int B, int Ttok, int nprefix,
                                   int D) {
    const long total = (long)B * nprefix * D;
    for (long t = blockIdx.x * (long)blockDim.x + threadIdx.x; t < total; t += (long)gridDim.x * blockDim.x) {
        const int d = (int)(t % D);
        const int pi = (int)((t / D) % nprefix);
        const int b = (int)(t / ((long)D * nprefix));
        const float v = vec[pi * D + d];
        if constexpr (sizeof(T) == 4) x[((long)b * Ttok + pi) * D + d] = v;
        else x[((long)b * Ttok + pi) * D + d] = __float2bfloat16_rn(v);
    }
}
// masked patches are REPLACED by mask_token (encoders/vision_transformer.py:195); idx = flat index into [B*HW]
template <typename T>
__global__ void mask_token_kernel(T* __restrict__ x, const float* __restrict__ tok, const long long* __restrict__ idx,
                                  int n, int HW, int Ttok, int prefix, int D) {
    const long total = (long)n * D;
    for (long t = blockIdx.x * (long)blockDim.x + threadIdx.x; t < total; t += (long)gridDim.x * blockDim.x) {
        const int d = (int)(t % D);
        const long long f = idx[t / D];
        const long row = (f / HW) * Ttok + prefix + f % HW;
        if constexpr (sizeof(T) == 4) x[row * D + d] = tok[d];
        else x[row * D + d] = __float2bfloat16_rn(tok[d]);
    }
}

// ------------------------------------------------------------------------------------------------ norms
// One warp per row.  RMSNorm (layers/normalization.py:17-22): y = (x * rsqrt(mean(x^2)+eps)).type_as(x) * w
// LayerNorm (nn.LayerNorm): y = (x-mean)*rsqrt(var+eps)*w + b.     Output: fp32 | bf16 | bf16x3 split [hi|hi|lo].
template <typename T>
__device__ __forceinline__ void load4(const T* p, float (&v)[4]);
template <>
__device__ __forceinline__ void load4<float>(const float* p, float (&v)[4]) {
    float4 t = *reinterpret_cast<const float4*>(p);
    v[0] = t.x, v[1] = t.y, v[2] = t.z, v[3] = t.w;
}
template <>
__device__ __forceinline__ void load4<__nv_bfloat16>(const __nv_bfloat16* p, float (&v)[4]) {
    uint2 t = *reinterpret_cast<const uint2*>(p);
    v[0] = bf16_lo(t.x), v[1] = bf16_hi(t.x), v[2] = bf16_lo(t.y), v[3] = bf16_hi(t.y);
}

enum { OUT_F32 = 0, OUT_BF16 = 1, OUT_SPLIT3 = 2 };

template <typename TIn, int MAXV>  // MAXV = max float4 groups per lane (D <= 128*MAXV)
__global__ void norm_fwd_kernel(const TIn* __restrict__ x, void* __restrict__ y, int y_mode,
                                const float* __restrict__ w, const float* __restrict__ b, float eps, int M, int D,
                                long ldx, float* __restrict__ rstd_out, float* __restrict__ mean_out, int is_ln) {
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (warp >= M) return;
    const TIn* xr = x + (long)warp * ldx;
    float v[MAXV][4];
    float s = 0.f;
#pragma unroll
    for (int g = 0; g < MAXV; ++g) {
        const int c = (g * 32 + lane) * 4;
        if (c < D) {
            load4<TIn>(xr + c, v[g]);
            s += is_ln ? (v[g][0] + v[g][1] + v[g][2] + v[g][3])
                       : (v[g][0] * v[g][0] + v[g][1] * v[g][1] + v[g][2] * v[g][2] + v[g][3] * v[g][3]);
        }
    }
    s = warp_sum(s);
    float mean = 0.f, rstd;
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
    if (lane == 0) {
        if (rstd_out) rstd_out[warp] = rstd;
        if (mean_out) mean_out[warp] = mean;
    }
#pragma unroll
    for (int g = 0; g < MAXV; ++g) {
        const int c = (g * 32 + lane) * 4;
        if (c < D) {
            const float4 w4 = __ldg(reinterpret_cast<const float4*>(w + c));
            float o[4];
            if (is_ln) {
                const float4 b4 = __ldg(reinterpret_cast<const float4*>(b + c));
                o[0] = (v[g][0] - mean) * rstd * w4.x + b4.x, o[1] = (v[g][1] - mean) * rstd * w4.y + b4.y;
                o[2] = (v[g][2] - mean) * rstd * w4.z + b4.z, o[3] = (v[g][3] - mean) * rstd * w4.w + b4.w;
            } else {
                float n0 = v[g][0] * rstd, n1 = v[g][1] * rstd, n2 = v[g][2] * rstd, n3 = v[g][3] * rstd;
                if constexpr (sizeof(TIn) == 2) {  // .type_as(x) before the weight multiply
                    n0 = bf16_round(n0), n1 = bf16_round(n1), n2 = bf16_round(n2), n3 = bf16_round(n3);
                }
                o[0] = n0 * w4.x, o[1] = n1 * w4.y, o[2] = n2 * w4.z, o[3] = n3 * w4.w;
            }
            if (y_mode == OUT_F32) {
                *reinterpret_cast<float4*>(reinterpret_cast<float*>(y) + (long)warp * D + c) =
                    make_float4(o[0], o[1], o[2], o[3]);
            } else if (y_mode == OUT_BF16) {
                uint2 t;
                t.x = pack_bf16x2(o[0], o[1]), t.y = pack_bf16x2(o[2], o[3]);
                *reinterpret_cast<uint2*>(reinterpret_cast<__nv_bfloat16*>(y) + (long)warp * D + c) = t;
            } else {
                float hi[4], lo[4];
#pragma unroll
                for (int i = 0; i < 4; ++i) hi[i] = bf16_round(o[i]), lo[i] = o[i] - hi[i];
                uint2 th, tl;
                th.x = pack_bf16x2(hi[0], hi[1]), th.y = pack_bf16x2(hi[2], hi[3]);
                tl.x = pack_bf16x2(lo[0], lo[1]), tl.y = pack_bf16x2(lo[2], lo[3]);
                __nv_bfloat16* yr = reinterpret_cast<__nv_bfloat16*>(y) + (long)warp * 3 * D;
                *reinterpret_cast<uint2*>(yr + c) = th;
                *reinterpret_cast<uint2*>(yr + D + c) = th;
                *reinterpret_cast<uint2*>(yr + 2 * D + c) = tl;
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------ bf16x3 split
// x fp32 [M][ldx] (K used) -> out bf16 [M][3K]:  which=0 (A side): [hi|hi|lo]   which=1 (B side): [hi|lo|hi]
// so that  A'·B'ᵀ = hi·hi + hi·lo + lo·hi  (error ~2^-16 relative; the dropped lo·lo term is 2^-18).
__global__ void split3_kernel(const float* __restrict__ x, __nv_bfloat16* __restrict__ out, long M, int K, long ldx,
                              int which) {
    const long total = M * (K / 4);
    for (long t = blockIdx.x * (long)blockDim.x + threadIdx.x; t < total; t += (long)gridDim.x * blockDim.x) {
        const long r = t / (K / 4);
        const int c = (int)(t % (K / 4)) * 4;
        const float4 v = *reinterpret_cast<const float4*>(x + r * ldx + c);
        const float f[4] = {v.x, v.y, v.z, v.w};
        float hi[4], lo[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) hi[i] = bf16_round(f[i]), lo[i] = f[i] - hi[i];
        uint2 th, tl;
        th.x = pack_bf16x2(hi[0], hi[1]), th.y = pack_bf16x2(hi[2], hi[3]);
        tl.x = pack_bf16x2(lo[0], lo[1]), tl.y = pack_bf16x2(lo[2], lo[3]);
        __nv_bfloat16* o = out + r * 3 * K + c;
        *reinterpret_cast<uint2*>(o) = th;
        *reinterpret_cast<uint2*>(o + K) = which ? tl : th;
        *reinterpret_cast<uint2*>(o + 2 * K) = which ? th : tl;
    }
}

// ------------------------------------------------------------------------------------------------ batched transpose
// in [B][R][C] -> out [B][C][R] with dtype conversion (latents (B,HW,64) <-> (B,64,H,W), modeling_vtp.py:395,
// pixel_decoder.py:141)
template <typename TI, typename TO>
__global__ void transpose_kernel(const TI* __restrict__ in, TO* __restrict__ out, int R, int C, long in_bstride,
                                 long out_bstride) {
    __shared__ float tile[32][33];
    const int b = blockIdx.z;
    const int r0 = blockIdx.y * 32, c0 = blockIdx.x * 32;
    const TI* ib = in + (long)b * in_bstride;
    TO* ob = out + (long)b * out_bstride;
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
        const int r = r0 + i, c = c0 + threadIdx.x;
        if (r < R && c < C) tile[i][threadIdx.x] = (float)ib[(long)r * C + c];
    }
    __syncthreads();
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
        const int c = c0 + i, r = r0 + threadIdx.x;
        if (r < R && c < C) ob[(long)c * R + r] = (TO)tile[threadIdx.x][i];
    }
}

// ------------------------------------------------------------------------------------------------ gather rows
// out[i][:] = in[idx[i]][:]   (iBOT masked-patch gather, vtp.py:432-439,470-473; text argmax pool)
template <typename TI, typename TO>
__global__ void gather_rows_kernel(const TI* __restrict__ in, TO* __restrict__ out, const long long* __restrict__ idx,
                                   int n, int D, long ld_in, long ld_out) {
    const long total = (long)n * D;
    for (long t = blockIdx.x * (long)blockDim.x + threadIdx.x; t < total; t += (long)gridDim.x * blockDim.x) {
        const int d = (int)(t % D);
        const long i = t / D;
        out[i * ld_out + d] = (TO)(float)in[idx[i] * ld_in + d];
    }
}


// ------------------------------------------------------------------------------------------------ batch-subset stochastic depth
// layers/block.py:201-233: a sub-layer runs on a random subset of the images only — `x[indices]` on the way in and
// `torch.index_add(x, 0, residual, indices, alpha = b / keep)` on the way out.  Image-granular (T token rows per index),
// 16-byte accesses; the indices of one call are distinct (a permutation prefix), so the add needs no atomics.
__global__ void gather_images_kernel(const float* __restrict__ x, float* __restrict__ out, const long long* __restrict__ idx,
                                     int n_img, int T, int D4, float alpha) {
    const long per = (long)T * D4, total = (long)n_img * per;
    for (long t = blockIdx.x * (long)blockDim.x + threadIdx.x; t < total; t += (long)gridDim.x * blockDim.x) {
        const long i = t / per, r = t - i * per;
        float4 v = reinterpret_cast<const float4*>(x)[idx[i] * per + r];
        v.x *= alpha, v.y *= alpha, v.z *= alpha, v.w *= alpha;
        reinterpret_cast<float4*>(out)[t] = v;
    }
}
template <typename TS>
__global__ void scatter_add_images_kernel(const TS* __restrict__ src, float* __restrict__ dst, const long long* __restrict__ idx,
                                          int n_img, int T, int D4, float alpha) {
    const long per = (long)T * D4, total = (long)n_img * per;
    for (long t = blockIdx.x * (long)blockDim.x + threadIdx.x; t < total; t += (long)gridDim.x * blockDim.x) {
        const long i = t / per, r = t - i * per;
        float s4[4];
        if constexpr (sizeof(TS) == 4) {
            const float4 v = reinterpret_cast<const float4*>(src)[t];
            s4[0] = v.x, s4[1] = v.y, s4[2] = v.z, s4[3] = v.w;
        } else {
            const uint2 v = reinterpret_cast<const uint2*>(src)[t];
            s4[0] = bf16_lo(v.x), s4[1] = bf16_hi(v.x), s4[2] = bf16_lo(v.y), s4[3] = bf16_hi(v.y);
        }
        float4* d = reinterpret_cast<float4*>(dst) + idx[i] * per + r;
        float4 o = *d;
        o.x = fmaf(alpha, s4[0], o.x), o.y = fmaf(alpha, s4[1], o.y), o.z = fmaf(alpha, s4[2], o.z), o.w = fmaf(alpha, s4[3], o.w);
        *d = o;
    }
}

// ------------------------------------------------------------------------------------------------ text embedding
// out[b*L + l][:] = emb[ids[b][l]][:] + pos[l][:]   (vtp_hf/modeling_vtp.py:297-298)
__global__ void embed_tokens_kernel(const long long* __restrict__ ids, const float* __restrict__ emb,
                                    const float* __restrict__ pos, float* __restrict__ out, long BL, int L, int D) {
    const long total = BL * (D / 4);
    for (long t = blockIdx.x * (long)blockDim.x + threadIdx.x; t < total; t += (long)gridDim.x * blockDim.x) {
        const long r = t / (D / 4);
        const int c = (int)(t % (D / 4)) * 4;
        const float4 e = __ldg(reinterpret_cast<const float4*>(emb + ids[r] * D + c));
        const float4 q = __ldg(reinterpret_cast<const float4*>(pos + (r % L) * D + c));
        *reinterpret_cast<float4*>(out + r * D + c) = make_float4(e.x + q.x, e.y + q.y, e.z + q.z, e.w + q.w);
    }
}

// ------------------------------------------------------------------------------------------------ L2 normalise
// y = x / max(||x||_2, eps) per row (F.normalize, vtp_hf/modeling_vtp.py:276,310; heads/dino_head.py:83-84).
// One warp per row; x fp32|bf16 [M][D], y fp32|bf16; optional norm_out [M] (saved for backward).
template <typename TI, typename TO>
__global__ void l2norm_kernel(const TI* __restrict__ x, TO* __restrict__ y, float* __restrict__ norm_out, int M, int D,
                              float eps) {
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (warp >= M) return;
    const TI* xr = x + (long)warp * D;
    float s = 0.f;
    for (int c = lane; c < D; c += 32) {
        const float v = (float)xr[c];
        s += v * v;
    }
    s = warp_sum(s);
    const float nrm = sqrtf(s);
    const float inv = 1.f / fmaxf(nrm, eps);
    if (lane == 0 && norm_out) norm_out[warp] = nrm;
    for (int c = lane; c < D; c += 32) y[(long)warp * D + c] = (TO)((float)xr[c] * inv);
}

static inline int grid_for(long total, int block) {
    long g = (total + block - 1) / block;
    long cap = (long)num_sms() * 16;
    return (int)(g < cap ? (g > 0 ? g : 1) : cap);
}

}  // namespace vtp

using namespace vtp;

extern "C" int vtp_patchify(const float* img, void* out, int out_dtype, int B, int C, int H, int W, int p,
                            vtp_stream_t st) {
    VTP_CHECK_ARG(img && out && B > 0 && C > 0, "patchify: bad args");
    VTP_CHECK_ARG(H % p == 0 && W % p == 0 && p % 4 == 0, "patchify: H,W must be multiples of p, p %% 4 == 0");
    VTP_CHECK_ARG((reinterpret_cast<uintptr_t>(img) & 15) == 0 && W % 4 == 0, "patchify: alignment");
    const long total4 = (long)B * C * H * W / 4;
    if (out_dtype == VTP_F32)
        patchify_kernel<float><<<grid_for(total4, 256), 256, 0, (cudaStream_t)st>>>(img, (float*)out, B, C, H, W, p, total4);
    else
        patchify_kernel<__nv_bfloat16>
            <<<grid_for(total4, 256), 256, 0, (cudaStream_t)st>>>(img, (__nv_bfloat16*)out, B, C, H, W, p, total4);
    VTP_LAUNCH_CHECK();
    return VTP_OK;
}

extern "C" int vtp_fill_prefix_tokens(void* x, int x_dtype, const float* vec, int B, int tokens, int nprefix, int D,
                                      vtp_stream_t st) {
    VTP_CHECK_ARG(x && vec && B > 0 && nprefix > 0 && nprefix <= tokens, "fill_prefix: bad args");
    const long total = (long)B * nprefix * D;
    if (x_dtype == VTP_F32)
        fill_prefix_kernel<float><<<grid_for(total, 256), 256, 0, (cudaStream_t)st>>>((float*)x, vec, B, tokens, nprefix, D);
    else
        fill_prefix_kernel<__nv_bfloat16>
            <<<grid_for(total, 256), 256, 0, (cudaStream_t)st>>>((__nv_bfloat16*)x, vec, B, tokens, nprefix, D);
    VTP_LAUNCH_CHECK();
    return VTP_OK;
}

extern "C" int vtp_apply_mask_tokens(void* x, int x_dtype, const float* mask_token, const int64_t* idx, int n, int HW,
                                     int tokens, int prefix, int D, vtp_stream_t st) {
    VTP_CHECK_ARG(x && mask_token && (idx || n == 0), "mask_tokens: bad args");
    if (n == 0) return VTP_OK;
    const long total = (long)n * D;
    if (x_dtype == VTP_F32)
        mask_token_kernel<float><<<grid_for(total, 256), 256, 0, (cudaStream_t)st>>>(
            (float*)x, mask_token, (const long long*)idx, n, HW, tokens, prefix, D);
    else
        mask_token_kernel<__nv_bfloat16><<<grid_for(total, 256), 256, 0, (cudaStream_t)st>>>(
            (__nv_bfloat16*)x, mask_token, (const long long*)idx, n, HW, tokens, prefix, D);
    VTP_LAUNCH_CHECK();
    return VTP_OK;
}

extern "C" int vtp_norm_fwd(const void* x, int x_dtype, long ldx, void* y, int y_mode, const float* w, const float* b,
                            float eps, int M, int D, float* rstd_out, float* mean_out, vtp_stream_t st) {
    VTP_CHECK_ARG(x && y && w && M > 0, "norm_fwd: bad args");
    VTP_CHECK_ARG(D % 4 == 0 && D <= 2048 && ldx % 4 == 0, "norm_fwd: D must be a multiple of 4 and <= 2048");
    VTP_CHECK_ARG(y_mode >= 0 && y_mode <= 2, "norm_fwd: bad y_mode");
    const int is_ln = b != nullptr;
    const int threads = 256, rows_per_block = threads / 32;
    const int grid = ceil_div(M, rows_per_block);
    cudaStream_t s = (cudaStream_t)st;
#define LAUNCH_NORM(T, MV) \
    norm_fwd_kernel<T, MV><<<grid, threads, 0, s>>>((const T*)x, y, y_mode, w, b, eps, M, D, ldx, rstd_out, mean_out, is_ln)
    if (x_dtype == VTP_F32) {
        if (D <= 512) LAUNCH_NORM(float, 4);
        else if (D <= 1024) LAUNCH_NORM(float, 8);
        else LAUNCH_NORM(float, 16);
    } else {
        if (D <= 512) LAUNCH_NORM(__nv_bfloat16, 4);
        else if (D <= 1024) LAUNCH_NORM(__nv_bfloat16, 8);
        else LAUNCH_NORM(__nv_bfloat16, 16);
    }
#undef LAUNCH_NORM
    VTP_LAUNCH_CHECK();
    return VTP_OK;
}

extern "C" int vtp_split3(const float* x, long ldx, void* out_bf16, long M, int K, int b_side, vtp_stream_t st) {
    VTP_CHECK_ARG(x && out_bf16 && M > 0 && K % 8 == 0 && ldx % 4 == 0, "split3: bad args (K %% 8 == 0)");
    split3_kernel<<<grid_for(M * (K / 4), 256), 256, 0, (cudaStream_t)st>>>(x, (__nv_bfloat16*)out_bf16, M, K, ldx,
                                                                            b_side);
    VTP_LAUNCH_CHECK();
    return VTP_OK;
}

extern "C" int vtp_transpose_batched(const void* in, int in_dtype, long in_bstride, void* out, int out_dtype,
                                     long out_bstride, int B, int R, int C, vtp_stream_t st) {
    VTP_CHECK_ARG(in && out && B > 0 && R > 0 && C > 0 && B <= 65535, "transpose: bad args");
    dim3 grid(ceil_div(C, 32), ceil_div(R, 32), B), block(32, 8);
    cudaStream_t s = (cudaStream_t)st;
    if (in_dtype == VTP_F32 && out_dtype == VTP_F32)
        transpose_kernel<float, float><<<grid, block, 0, s>>>((const float*)in, (float*)out, R, C, in_bstride, out_bstride);
    else if (in_dtype == VTP_F32)
        transpose_kernel<float, __nv_bfloat16><<<grid, block, 0, s>>>((const float*)in, (__nv_bfloat16*)out, R, C, in_bstride, out_bstride);
    else if (out_dtype == VTP_F32)
        transpose_kernel<__nv_bfloat16, float><<<grid, block, 0, s>>>((const __nv_bfloat16*)in, (float*)out, R, C, in_bstride, out_bstride);
    else
        transpose_kernel<__nv_bfloat16, __nv_bfloat16>
            <<<grid, block, 0, s>>>((const __nv_bfloat16*)in, (__nv_bfloat16*)out, R, C, in_bstride, out_bstride);
    VTP_LAUNCH_CHECK();
    return VTP_OK;
}

extern "C" int vtp_gather_rows(const void* in, int in_dtype, long ld_in, void* out, int out_dtype, long ld_out,
                               const int64_t* idx, int n, int D, vtp_stream_t st) {
    VTP_CHECK_ARG(in && out && (idx || n == 0), "gather_rows: bad args");
    if (n == 0) return VTP_OK;
    const long total = (long)n * D;
    cudaStream_t s = (cudaStream_t)st;
    const int g = grid_for(total, 256);
    const long long* ix = (const long long*)idx;
    if (in_dtype == VTP_F32 && out_dtype == VTP_F32)
        gather_rows_kernel<float, float><<<g, 256, 0, s>>>((const float*)in, (float*)out, ix, n, D, ld_in, ld_out);
    else if (in_dtype == VTP_F32)
        gather_rows_kernel<float, __nv_bfloat16>
            <<<g, 256, 0, s>>>((const float*)in, (__nv_bfloat16*)out, ix, n, D, ld_in, ld_out);
    else if (out_dtype == VTP_F32)
        gather_rows_kernel<__nv_bfloat16, float>
            <<<g, 256, 0, s>>>((const __nv_bfloat16*)in, (float*)out, ix, n, D, ld_in, ld_out);
    else
        gather_rows_kernel<__nv_bfloat16, __nv_bfloat16>
            <<<g, 256, 0, s>>>((const __nv_bfloat16*)in, (__nv_bfloat16*)out, ix, n, D, ld_in, ld_out);
    VTP_LAUNCH_CHECK();
    return VTP_OK;
}

extern "C" int vtp_gather_images(const float* x, float* out, const int64_t* img_idx, int n_img, int T, int D, float alpha,
                                 vtp_stream_t st) {
    VTP_CHECK_ARG(x && out && (img_idx || n_img == 0) && T > 0 && D > 0 && D % 4 == 0, "gather_images: bad args (D %% 4 == 0)");
    if (n_img == 0) return VTP_OK;
    gather_images_kernel<<<grid_for((long)n_img * T * (D / 4), 256), 256, 0, (cudaStream_t)st>>>(
        x, out, (const long long*)img_idx, n_img, T, D / 4, alpha);
    VTP_LAUNCH_CHECK();
    return VTP_OK;
}

extern "C" int vtp_scatter_add_images(const void* src, int src_dtype, float* dst, const int64_t* img_idx, int n_img, int T,
                                      int D, float alpha, vtp_stream_t st) {
    VTP_CHECK_ARG(src && dst && (img_idx || n_img == 0) && T > 0 && D > 0 && D % 4 == 0, "scatter_add_images: bad args");
    VTP_CHECK_ARG(src_dtype == VTP_F32 || src_dtype == VTP_BF16, "scatter_add_images: bad src dtype");
    if (n_img == 0) return VTP_OK;
    const int g = grid_for((long)n_img * T * (D / 4), 256);
    if (src_dtype == VTP_F32)
        scatter_add_images_kernel<float><<<g, 256, 0, (cudaStream_t)st>>>((const float*)src, dst, (const long long*)img_idx, n_img,
                                                                       T, D / 4, alpha);
    else
        scatter_add_images_kernel<__nv_bfloat16><<<g, 256, 0, (cudaStream_t)st>>>(
            (const __nv_bfloat16*)src, dst, (const long long*)img_idx, n_img, T, D / 4, alpha);
    VTP_LAUNCH_CHECK();
    return VTP_OK;
}

extern "C" int vtp_embed_tokens(const int64_t* ids, const float* emb, const float* pos, float* out, long BL, int L, int D,
                                vtp_stream_t st) {
    VTP_CHECK_ARG(ids && emb && pos && out && BL > 0 && D % 4 == 0, "embed_tokens: bad args");
    embed_tokens_kernel<<<grid_for(BL * (D / 4), 256), 256, 0, (cudaStream_t)st>>>((const long long*)ids, emb, pos, out,
                                                                                   BL, L, D);
    VTP_LAUNCH_CHECK();
    return VTP_OK;
}

extern "C" int vtp_l2norm_fwd(const void* x, int x_dtype, void* y, int y_dtype, float* norm_out, int M, int D, float eps,
                              vtp_stream_t st) {
    VTP_CHECK_ARG(x && y && M > 0 && D > 0, "l2norm_fwd: bad args");
    const int grid = ceil_div(M, 8);
    cudaStream_t s = (cudaStream_t)st;
    if (x_dtype == VTP_F32 && y_dtype == VTP_F32)
        l2norm_kernel<float, float><<<grid, 256, 0, s>>>((const float*)x, (float*)y, norm_out, M, D, eps);
    else if (x_dtype == VTP_F32)
        l2norm_kernel<float, __nv_bfloat16><<<grid, 256, 0, s>>>((const float*)x, (__nv_bfloat16*)y, norm_out, M, D, eps);
    else if (y_dtype == VTP_F32)
        l2norm_kernel<__nv_bfloat16, float><<<grid, 256, 0, s>>>((const __nv_bfloat16*)x, (float*)y, norm_out, M, D, eps);
    else
        l2norm_kernel<__nv_bfloat16, __nv_bfloat16>
            <<<grid, 256, 0, s>>>((const __nv_bfloat16*)x, (__nv_bfloat16*)y, norm_out, M, D, eps);
    VTP_LAUNCH_CHECK();
    return VTP_OK;
}

// ------------------------------------------------------------------------------------------------ SwiGLU gate / RoPE
// Stand-alone (full-occupancy) versions of the two heaviest GEMM epilogues: at K = 384 the GEMM's 8 epilogue warps are
// instruction / latency bound on the RoPE arithmetic, a 64-warp/SM elementwise pass is not.
namespace vtp {
// pre bf16 [M][2Hs] (8-interleaved x1|x2) -> hid bf16 [M][Hs] = round(round(silu(x1)) * x2)   (layers/ffn.py:77-81)
__global__ void swiglu_fwd_kernel(const __nv_bfloat16* __restrict__ pre, __nv_bfloat16* __restrict__ hid, long M, int Hs) {
    const int G = Hs / 8;
    const long total = M * G;
    for (long t = blockIdx.x * (long)blockDim.x + threadIdx.x; t < total; t += (long)gridDim.x * blockDim.x) {
        const long row = t / G;
        const int g = (int)(t % G);
        const uint4 a = *reinterpret_cast<const uint4*>(pre + row * 2 * Hs + 16 * g);
        const uint4 b = *reinterpret_cast<const uint4*>(pre + row * 2 * Hs + 16 * g + 8);
        const uint32_t aw[4] = {a.x, a.y, a.z, a.w}, bw[4] = {b.x, b.y, b.z, b.w};
        uint32_t o[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const float x1l = bf16_lo(aw[k]), x1h = bf16_hi(aw[k]), x2l = bf16_lo(bw[k]), x2h = bf16_hi(bw[k]);
            const float sl = bf16_round(__fdividef(x1l, 1.f + __expf(-x1l))), sh = bf16_round(__fdividef(x1h, 1.f + __expf(-x1h)));
            o[k] = pack_bf16x2(sl * x2l, sh * x2h);
        }
        *reinterpret_cast<uint4*>(hid + row * Hs + 8 * g) = make_uint4(o[0], o[1], o[2], o[3]);
    }
}

// in-place axial RoPE on the q,k parts of a packed bf16 qkv buffer [B*T][3D] (layers/attention.py:70-89, bf16 arithmetic
// with a rounding after every op); one thread = one (row, head, q|k) 64-vector half pair chunk of 8+8 elements
__global__ void rope_fwd_kernel(__nv_bfloat16* __restrict__ qkv, const __nv_bfloat16* __restrict__ sin_,
                                const __nv_bfloat16* __restrict__ cos_, long rows, int T, int prefix, int D) {
    const int H2 = 2 * D / 64;  // q and k heads
    const long total = rows * H2 * 4;
    for (long t = blockIdx.x * (long)blockDim.x + threadIdx.x; t < total; t += (long)gridDim.x * blockDim.x) {
        const int c8 = (int)(t & 3) * 8;
        const int hh = (int)((t >> 2) % H2);
        const long row = t / (4L * H2);
        const int pos = (int)(row % T) - prefix;
        if (pos < 0) continue;
        __nv_bfloat16* base = qkv + row * 3 * D + hh * 64 + c8;
        const uint4 lo = *reinterpret_cast<const uint4*>(base), hi = *reinterpret_cast<const uint4*>(base + 32);
        const uint4 sl = __ldg(reinterpret_cast<const uint4*>(sin_ + (long)pos * 64 + c8));
        const uint4 cl = __ldg(reinterpret_cast<const uint4*>(cos_ + (long)pos * 64 + c8));
        const uint4 sh = __ldg(reinterpret_cast<const uint4*>(sin_ + (long)pos * 64 + 32 + c8));
        const uint4 ch = __ldg(reinterpret_cast<const uint4*>(cos_ + (long)pos * 64 + 32 + c8));
        const uint32_t lw[4] = {lo.x, lo.y, lo.z, lo.w}, hw[4] = {hi.x, hi.y, hi.z, hi.w};
        const uint32_t slw[4] = {sl.x, sl.y, sl.z, sl.w}, clw[4] = {cl.x, cl.y, cl.z, cl.w};
        const uint32_t shw[4] = {sh.x, sh.y, sh.z, sh.w}, chw[4] = {ch.x, ch.y, ch.z, ch.w};
        uint32_t ol[4], oh[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            float rl[2], rh[2];
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const float a = e ? bf16_hi(lw[k]) : bf16_lo(lw[k]), b = e ? bf16_hi(hw[k]) : bf16_lo(hw[k]);
                const float s0 = e ? bf16_hi(slw[k]) : bf16_lo(slw[k]), c0 = e ? bf16_hi(clw[k]) : bf16_lo(clw[k]);
                const float s1 = e ? bf16_hi(shw[k]) : bf16_lo(shw[k]), c1 = e ? bf16_hi(chw[k]) : bf16_lo(chw[k]);
                rl[e] = bf16_round(a * c0) + bf16_round((-b) * s0);
                rh[e] = bf16_round(b * c1) + bf16_round(a * s1);
            }
            ol[k] = pack_bf16x2(rl[0], rl[1]), oh[k] = pack_bf16x2(rh[0], rh[1]);
        }
        *reinterpret_cast<uint4*>(base) = make_uint4(ol[0], ol[1], ol[2], ol[3]);
        *reinterpret_cast<uint4*>(base + 32) = make_uint4(oh[0], oh[1], oh[2], oh[3]);
    }
}
}  // namespace vtp

extern "C" int vtp_swiglu_fwd(const void* pre, void* hid, long M, int Hs, vtp_stream_t st) {
    VTP_CHECK_ARG(pre && hid && M > 0 && Hs % 8 == 0, "swiglu_fwd: bad args");
    vtp::swiglu_fwd_kernel<<<vtp::grid_for(M * (Hs / 8), 256), 256, 0, (cudaStream_t)st>>>((const __nv_bfloat16*)pre,
                                                                                           (__nv_bfloat16*)hid, M, Hs);
    VTP_LAUNCH_CHECK();
    return VTP_OK;
}

extern "C" int vtp_rope_fwd(void* qkv, const void* sin_, const void* cos_, long rows, int T, int prefix, int D,
                            vtp_stream_t st) {
    VTP_CHECK_ARG(qkv && sin_ && cos_ && rows > 0 && T > 0 && D % 64 == 0, "rope_fwd: bad args");
    vtp::rope_fwd_kernel<<<vtp::grid_for(rows * (2 * D / 64) * 4, 256), 256, 0, (cudaStream_t)st>>>(
        (__nv_bfloat16*)qkv, (const __nv_bfloat16*)sin_, (const __nv_bfloat16*)cos_, rows, T, prefix, D);
    VTP_LAUNCH_CHECK();
    return VTP_OK;
}
