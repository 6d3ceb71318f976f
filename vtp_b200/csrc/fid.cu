// vtp_b200 — the Fréchet Inception Distance of pytorch-fid (fid_score.calculate_fid_given_paths, dims = 2048) on the
// device.  The 94 convolutions of the Inception network are vtp_gemm_bf16 on bf16x3 operands with fp32 output; this
// file holds the passes around them:
//   fid_resize   uint8 NHWC -> ToTensor (x * fl(1/255), torch's CUDA division by a scalar), bilinear resize to 299x299
//                with torch's upsample_bilinear2d arithmetic, then 2x - 1: the network input, fp32 NHWC
//   fid_im2col3  any (kh, kw, stride, pad) of the network -> the [hi|hi|lo] bf16x3 A operand of the conv GEMM
//   fid_pool     3x3 max / average pools into a channel slice of a block's concatenated output
//   fid_moments  spatial mean of the last block -> fp64 sums S1 = Σ f, S2 = Σ f fᵀ (upper triangle), n
// No atomics anywhere: repeated runs are bit-identical.
#include "host.h"
#include "ptx.cuh"

namespace vtp {

constexpr int FID_SIZE = 299;

// torch/aten/src/ATen/native/cuda/UpSampleBilinear2d.cu (upsample_bilinear2d_out_frame, align_corners = False), per
// output pixel and channel, written as the same expressions so that the compiler contracts them as in torch's build:
//   src = scale * (dst + 0.5) - 0.5, clamped at 0;  i = (int)src;  lambda1 = src - i;  lambda0 = 1 - lambda1
//   val = h0 * (w0 * v00 + w1 * v01) + h1 * (w0 * v10 + w1 * v11)
// The source values are fl(u * fl(1/255)), rounded before they enter the blend (a separate torch kernel).  The
// resized value then goes through 2 * x (exact) and - 1 (one rounding).  When H = W = 299 torch copies the input.
__global__ void __launch_bounds__(256) fid_resize_kernel(const uint8_t* __restrict__ u8, int B, int H, int W, float rh,
                                                         float rw, float* __restrict__ out) {
    const long total = (long)B * FID_SIZE * FID_SIZE;
    const float inv255 = 1.0f / 255.0f;
    const bool copy = H == FID_SIZE && W == FID_SIZE;
    for (long t = blockIdx.x * (long)blockDim.x + threadIdx.x; t < total; t += (long)gridDim.x * blockDim.x) {
        const int w2 = (int)(t % FID_SIZE), h2 = (int)((t / FID_SIZE) % FID_SIZE);
        const long b = t / (FID_SIZE * FID_SIZE);
        const uint8_t* img = u8 + b * H * W * 3;
        float v[3];
        if (copy) {
#pragma unroll
            for (int c = 0; c < 3; ++c) v[c] = __fmul_rn((float)img[((long)h2 * W + w2) * 3 + c], inv255);
        } else {
            float h1r = rh * (h2 + 0.5f) - 0.5f;
            h1r = h1r < 0.f ? 0.f : h1r;
            const int h1 = (int)h1r;
            const int h1p = (h1 < H - 1) ? 1 : 0;
            const float h1lambda = h1r - h1;
            const float h0lambda = 1.f - h1lambda;
            float w1r = rw * (w2 + 0.5f) - 0.5f;
            w1r = w1r < 0.f ? 0.f : w1r;
            const int w1 = (int)w1r;
            const int w1p = (w1 < W - 1) ? 1 : 0;
            const float w1lambda = w1r - w1;
            const float w0lambda = 1.f - w1lambda;
            const uint8_t* p00 = img + ((long)h1 * W + w1) * 3;
            const uint8_t* p01 = p00 + w1p * 3;
            const uint8_t* p10 = p00 + (long)h1p * W * 3;
            const uint8_t* p11 = p10 + w1p * 3;
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                const float a = __fmul_rn((float)p00[c], inv255), bq = __fmul_rn((float)p01[c], inv255);
                const float cq = __fmul_rn((float)p10[c], inv255), d = __fmul_rn((float)p11[c], inv255);
                v[c] = h0lambda * (w0lambda * a + w1lambda * bq) + h1lambda * (w0lambda * cq + w1lambda * d);
            }
        }
        float* o = out + t * 3;
#pragma unroll
        for (int c = 0; c < 3; ++c) o[c] = __fadd_rn(__fmul_rn(2.f, v[c]), -1.f);
    }
}

// Output row m = (b*Ho + ho)*Wo + wo of the A operand [M][taps*3C]; tap t = dy*kw + dx reads input pixel
// (ho*s - ph + dy, wo*s - pw + dx), zero outside the image.  Per tap the row holds [hi | hi | lo] of the C channels
// (hi = bf16(x), lo = bf16(x - hi)), against the [hi | lo | hi] per-tap weights of vtp_split3(b_side = 1).
// One thread per (row, tap, 4 channels).
__global__ void __launch_bounds__(256) fid_im2col3_kernel(const float* __restrict__ in, int H, int W, int C, long ld_in,
                                                          int Ho, int Wo, int kh, int kw, int s, int ph, int pw, long M,
                                                          __nv_bfloat16* __restrict__ out) {
    const int C4 = C / 4, taps = kh * kw;
    const long K3 = (long)taps * 3 * C;
    const long total = M * taps * C4;
    for (long t = blockIdx.x * (long)blockDim.x + threadIdx.x; t < total; t += (long)gridDim.x * blockDim.x) {
        const int c = (int)(t % C4) * 4;
        const long r = t / C4;
        const int tap = (int)(r % taps);
        const long m = r / taps;
        const int wo = (int)(m % Wo), ho = (int)((m / Wo) % Ho);
        const long b = m / ((long)Wo * Ho);
        const int hi_ = ho * s - ph + tap / kw, wi = wo * s - pw + tap % kw;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (hi_ >= 0 && hi_ < H && wi >= 0 && wi < W)
            v = __ldg(reinterpret_cast<const float4*>(in + ((b * H + hi_) * W + wi) * ld_in + c));
        const float f[4] = {v.x, v.y, v.z, v.w};
        float h[4], l[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) h[i] = bf16_round(f[i]), l[i] = f[i] - h[i];
        uint2 th, tl;
        th.x = pack_bf16x2(h[0], h[1]), th.y = pack_bf16x2(h[2], h[3]);
        tl.x = pack_bf16x2(l[0], l[1]), tl.y = pack_bf16x2(l[2], l[3]);
        __nv_bfloat16* o = out + m * K3 + (long)tap * 3 * C + c;
        *reinterpret_cast<uint2*>(o) = th;
        *reinterpret_cast<uint2*>(o + C) = th;
        *reinterpret_cast<uint2*>(o + 2 * C) = tl;
    }
}

// The 3-channel stem (Conv2d_1a_3x3): k = tap*3 + c (27 values, padded to 32), row = [hi(32) | hi(32) | lo(32)], as
// vtp_lpips_prep3 lays out conv1_1 of the VGG.  One thread per output row.
__global__ void __launch_bounds__(128) fid_im2col3_stem_kernel(const float* __restrict__ in, int H, int W, long ld_in,
                                                               int Ho, int Wo, int s, int ph, int pw, long M,
                                                               __nv_bfloat16* __restrict__ out) {
    for (long m = blockIdx.x * (long)blockDim.x + threadIdx.x; m < M; m += (long)gridDim.x * blockDim.x) {
        const int wo = (int)(m % Wo), ho = (int)((m / Wo) % Ho);
        const long b = m / ((long)Wo * Ho);
        float vals[32];
#pragma unroll
        for (int tap = 0; tap < 9; ++tap) {
            const int hh = ho * s - ph + tap / 3, ww = wo * s - pw + tap % 3;
            const bool ok = hh >= 0 && hh < H && ww >= 0 && ww < W;
            const float* p = in + ((b * H + hh) * W + ww) * ld_in;
#pragma unroll
            for (int c = 0; c < 3; ++c) vals[tap * 3 + c] = ok ? __ldg(p + c) : 0.f;
        }
#pragma unroll
        for (int i = 27; i < 32; ++i) vals[i] = 0.f;
        uint32_t hi[16], lo[16];
#pragma unroll
        for (int i = 0; i < 16; ++i) {
            const float h0 = bf16_round(vals[2 * i]), h1 = bf16_round(vals[2 * i + 1]);
            hi[i] = pack_bf16x2(h0, h1);
            lo[i] = pack_bf16x2(vals[2 * i] - h0, vals[2 * i + 1] - h1);
        }
        uint4* o = reinterpret_cast<uint4*>(out + m * 96);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            o[i] = make_uint4(hi[4 * i], hi[4 * i + 1], hi[4 * i + 2], hi[4 * i + 3]);
            o[4 + i] = o[i];
            o[8 + i] = make_uint4(lo[4 * i], lo[4 * i + 1], lo[4 * i + 2], lo[4 * i + 3]);
        }
    }
}

// 3x3 pools on fp32 NHWC, one thread per (output pixel, 4 channels), the window walked row by row:
//   mode 0  max, stride 2, no padding;  mode 1  max, stride 1, pad 1;  mode 2  average, stride 1, pad 1,
//   count_include_pad = False (the sum of the in-image taps divided by their count).
// Max follows torch's rule (a NaN tap wins; padding never does).
__global__ void __launch_bounds__(256) fid_pool_kernel(const float* __restrict__ in, int H, int W, int C, long ld_in, int Ho,
                                                       int Wo, int mode, long P, float* __restrict__ out, long ld_out) {
    const int C4 = C / 4, s = mode == 0 ? 2 : 1, pad = mode == 0 ? 0 : 1;
    const long total = P * C4;
    for (long t = blockIdx.x * (long)blockDim.x + threadIdx.x; t < total; t += (long)gridDim.x * blockDim.x) {
        const int c = (int)(t % C4) * 4;
        const long pix = t / C4;
        const int wo = (int)(pix % Wo), ho = (int)((pix / Wo) % Ho);
        const long b = pix / ((long)Wo * Ho);
        const int h0 = max(ho * s - pad, 0), h1 = min(ho * s - pad + 3, H);
        const int w0 = max(wo * s - pad, 0), w1 = min(wo * s - pad + 3, W);
        float acc[4];
        const float init = mode == 2 ? 0.f : -INFINITY;
#pragma unroll
        for (int i = 0; i < 4; ++i) acc[i] = init;
        for (int h = h0; h < h1; ++h)
            for (int w = w0; w < w1; ++w) {
                const float4 v = __ldg(reinterpret_cast<const float4*>(in + ((b * H + h) * W + w) * ld_in + c));
                const float f[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    if (mode == 2) acc[i] = __fadd_rn(acc[i], f[i]);
                    else if (f[i] > acc[i] || f[i] != f[i]) acc[i] = f[i];
                }
            }
        if (mode == 2) {
            const float cnt = (float)((h1 - h0) * (w1 - w0));
#pragma unroll
            for (int i = 0; i < 4; ++i) acc[i] = __fdiv_rn(acc[i], cnt);
        }
        *reinterpret_cast<float4*>(out + pix * ld_out + c) = make_float4(acc[0], acc[1], acc[2], acc[3]);
    }
}

// grid: one CTA per 64x64 tile (ti <= tj) of the upper triangle of S2, 256 threads.  Each CTA walks the images in order:
// threads 0..63 form the spatial means of the tile's row channels, 64..127 of its column channels (each one channel,
// summed over the P pixels in ascending order in fp32 and divided by P, so every CTA forms the same value), then each
// thread adds its 4x4 block of products to fp64 registers (an fp32 x fp32 product is exact in fp64).  Images at or
// above *rows are not accumulated; diagonal CTAs also write the features of every image (feat may be null) and S1.
__global__ void __launch_bounds__(256) fid_moments_kernel(const float* __restrict__ x, int B, int P, int D,
                                                          const int* __restrict__ rows_p, float* __restrict__ feat,
                                                          double* __restrict__ S2, double* __restrict__ S1,
                                                          double* __restrict__ n) {
    __shared__ float fs[128];
    const int T = D / 64, tid = threadIdx.x;
    int ti = 0, rem = blockIdx.x;
    while (rem >= T - ti) rem -= T - ti, ++ti;
    const int tj = ti + rem;
    const bool diag = ti == tj;
    const int rows = min(max(*rows_p, 0), B);
    const int nb = (diag && feat) ? B : rows;
    const int ch = tid < 64 ? ti * 64 + tid : tj * 64 + (tid - 64);
    const float invP = 1.f / (float)P;
    double acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.0;
    double s1 = 0.0;
    const int r4 = (tid >> 4) * 4, c4 = (tid & 15) * 4;
    for (int b = 0; b < nb; ++b) {
        if (tid < 128) {
            const float* p = x + (long)b * P * D + ch;
            float sum = 0.f;
#pragma unroll 16
            for (int q = 0; q < P; ++q) sum = __fadd_rn(sum, __ldg(p + (long)q * D));
            fs[tid] = __fmul_rn(sum, invP);
        }
        __syncthreads();
        if (diag && feat && tid < 64) feat[(long)b * D + ch] = fs[tid];
        if (b < rows) {
            if (diag && tid < 64) s1 += (double)fs[tid];
            double a[4], c[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) a[i] = (double)fs[r4 + i], c[i] = (double)fs[64 + c4 + i];
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fma(a[i], c[j], acc[i][j]);
        }
        __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) S2[(long)(ti * 64 + r4 + i) * D + tj * 64 + c4 + j] += acc[i][j];
    if (diag && tid < 64) S1[ti * 64 + tid] += s1;
    if (blockIdx.x == 0 && tid == 0) n[0] += (double)rows;
}

static inline int fid_grid(long n, int block) {
    long g = (n + block - 1) / block;
    long cap = (long)num_sms() * 16;
    return (int)(g < 1 ? 1 : (g < cap ? g : cap));
}

}  // namespace vtp

using namespace vtp;

extern "C" int vtp_fid_resize(const uint8_t* u8, int B, int H, int W, float* out, vtp_stream_t st) {
    VTP_CHECK_ARG(u8 && out && B > 0 && H > 0 && W > 0, "fid_resize: bad args");
    const float rh = (float)H / (float)FID_SIZE, rw = (float)W / (float)FID_SIZE;  // torch: (float)in / out on the host
    fid_resize_kernel<<<fid_grid((long)B * FID_SIZE * FID_SIZE, 256), 256, 0, (cudaStream_t)st>>>(u8, B, H, W, rh, rw, out);
    VTP_LAUNCH_CHECK();
    return VTP_OK;
}

extern "C" int vtp_fid_im2col3(const float* in, long ld_in, int c0, int B, int H, int W, int C, int kh, int kw, int stride,
                               int ph, int pw, void* out_bf16, vtp_stream_t st) {
    VTP_CHECK_ARG(in && out_bf16 && B > 0 && H > 0 && W > 0 && C > 0 && kh > 0 && kw > 0 && stride > 0 && ph >= 0 &&
                      pw >= 0 && c0 >= 0 && c0 + C <= ld_in,
                  "fid_im2col3: bad args");
    const int Ho = (H + 2 * ph - kh) / stride + 1, Wo = (W + 2 * pw - kw) / stride + 1;
    VTP_CHECK_ARG(H + 2 * ph >= kh && W + 2 * pw >= kw, "fid_im2col3: %dx%d kernel larger than the padded %dx%d input", kh, kw,
                  H, W);
    VTP_CHECK_ARG(((uintptr_t)out_bf16 & 15) == 0, "fid_im2col3: out must be 16-byte aligned");
    const long M = (long)B * Ho * Wo;
    cudaStream_t stream = (cudaStream_t)st;
    if (C == 3) {
        VTP_CHECK_ARG(kh == 3 && kw == 3, "fid_im2col3: the 3-channel stem takes 3x3 kernels only");
        fid_im2col3_stem_kernel<<<fid_grid(M, 128), 128, 0, stream>>>(in + c0, H, W, ld_in, Ho, Wo, stride, ph, pw, M,
                                                                      (__nv_bfloat16*)out_bf16);
    } else {
        VTP_CHECK_ARG(C % 4 == 0 && ld_in % 4 == 0 && c0 % 4 == 0 && ((uintptr_t)in & 15) == 0,
                      "fid_im2col3: C, ld_in and c0 must be multiples of 4 (C = 3: the stem) and in 16-byte aligned");
        fid_im2col3_kernel<<<fid_grid(M * kh * kw * (C / 4), 256), 256, 0, stream>>>(
            in + c0, H, W, C, ld_in, Ho, Wo, kh, kw, stride, ph, pw, M, (__nv_bfloat16*)out_bf16);
    }
    VTP_LAUNCH_CHECK();
    return VTP_OK;
}

extern "C" int vtp_fid_pool(const float* in, long ld_in, int B, int H, int W, int C, int mode, float* out, long ld_out, int c0,
                            vtp_stream_t st) {
    VTP_CHECK_ARG(in && out && B > 0 && H > 0 && W > 0 && C > 0 && mode >= 0 && mode <= 2, "fid_pool: bad args");
    VTP_CHECK_ARG(C % 4 == 0 && ld_in % 4 == 0 && ld_out % 4 == 0 && c0 % 4 == 0 && C <= ld_in && c0 >= 0 && c0 + C <= ld_out &&
                      ((uintptr_t)in & 15) == 0 && ((uintptr_t)out & 15) == 0,
                  "fid_pool: C, ld_in, ld_out and c0 must be multiples of 4, the slice inside ld_out, pointers 16-byte aligned");
    VTP_CHECK_ARG(mode != 0 || (H >= 3 && W >= 3), "fid_pool: stride-2 pool needs H, W >= 3");
    const int Ho = mode == 0 ? (H - 3) / 2 + 1 : H, Wo = mode == 0 ? (W - 3) / 2 + 1 : W;
    const long P = (long)B * Ho * Wo;
    fid_pool_kernel<<<fid_grid(P * (C / 4), 256), 256, 0, (cudaStream_t)st>>>(in, H, W, C, ld_in, Ho, Wo, mode, P, out + c0,
                                                                               ld_out);
    VTP_LAUNCH_CHECK();
    return VTP_OK;
}

extern "C" int vtp_fid_moments(const float* x, int B, int P, int D, const int* rows, float* feat, double* S2, double* S1,
                               double* n, vtp_stream_t st) {
    VTP_CHECK_ARG(x && rows && S2 && S1 && n && B > 0 && P > 0 && D > 0 && D % 64 == 0, "fid_moments: bad args (D %% 64)");
    const int T = D / 64;
    fid_moments_kernel<<<T * (T + 1) / 2, 256, 0, (cudaStream_t)st>>>(x, B, P, D, rows, feat, S2, S1, n);
    VTP_LAUNCH_CHECK();
    return VTP_OK;
}
