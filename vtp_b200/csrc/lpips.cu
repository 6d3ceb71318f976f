// vtp_b200 — LPIPS perceptual loss (utils/lpips.py:61-171) forward + gradient w.r.t. the reconstructed image.
// The 13 VGG16 3x3 convolutions (and their dgrads) run on the wgmma GEMM in implicit-conv mode (gemm.cu, conv_C > 0);
// this file holds the HBM-bound pieces around them, all on NHWC bf16 activations:
//   lpips_prep      ScalingLayer (lpips.py:103-114) + im2col of the 3-channel input (K = 27 -> 32) for conv1_1
//   maxpool2_fwd    nn.MaxPool2d(2,2)
//   pool_relu_bwd   gradient routing of MaxPool2d(2,2) fused with the tap gradient add and the ReLU mask
//   lpips_tap       per-pixel unit-normalise, squared difference, 1x1 "lin" weights, spatial mean (lpips.py:88-100,
//                   169-175): loss value + gradient w.r.t. the reconstructed-image features
//   lpips_img_grad  col2im of the conv1_1 input gradient + ScalingLayer backward -> d(image) fp32 NCHW
#include "host.h"
#include "ptx.cuh"

namespace vtp {

__constant__ float LP_SHIFT[3] = {-0.030f, -0.088f, -0.188f};
__constant__ float LP_SCALE[3] = {0.458f, 0.448f, 0.450f};

template <typename TI>
__global__ void lpips_prep_kernel(const TI* __restrict__ img, __nv_bfloat16* __restrict__ out, int B, int H, int W) {
    const long P = (long)B * H * W;
    for (long pix = blockIdx.x * (long)blockDim.x + threadIdx.x; pix < P; pix += (long)gridDim.x * blockDim.x) {
        const int w = (int)(pix % W), h = (int)((pix / W) % H);
        const long b = pix / ((long)W * H);
        uint32_t pk[16];
        float vals[32];
#pragma unroll
        for (int tap = 0; tap < 9; ++tap) {
            const int hh = h + tap / 3 - 1, ww = w + tap % 3 - 1;
            const bool in = hh >= 0 && hh < H && ww >= 0 && ww < W;
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                float v = 0.f;
                if (in) v = ((float)img[((b * 3 + c) * H + hh) * W + ww] - LP_SHIFT[c]) / LP_SCALE[c];
                vals[tap * 3 + c] = v;
            }
        }
#pragma unroll
        for (int i = 27; i < 32; ++i) vals[i] = 0.f;
#pragma unroll
        for (int i = 0; i < 16; ++i) pk[i] = pack_bf16x2(vals[2 * i], vals[2 * i + 1]);
        uint4* o = reinterpret_cast<uint4*>(out + pix * 32);
#pragma unroll
        for (int i = 0; i < 4; ++i) o[i] = make_uint4(pk[4 * i], pk[4 * i + 1], pk[4 * i + 2], pk[4 * i + 3]);
    }
}

// x [B][H][W][C] -> y [B][H/2][W/2][C], 8 channels per thread
__global__ void maxpool2_fwd_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ y, int B, int H, int W,
                                    int C) {
    const int Ho = H / 2, Wo = W / 2, C8 = C / 8;
    const long total = (long)B * Ho * Wo * C8;
    for (long t = blockIdx.x * (long)blockDim.x + threadIdx.x; t < total; t += (long)gridDim.x * blockDim.x) {
        const int c = (int)(t % C8) * 8;
        const long pix = t / C8;
        const int wo = (int)(pix % Wo), ho = (int)((pix / Wo) % Ho);
        const long b = pix / ((long)Wo * Ho);
        const __nv_bfloat16* p0 = x + ((b * H + 2 * ho) * W + 2 * wo) * C + c;
        const uint4 a = *reinterpret_cast<const uint4*>(p0), bq = *reinterpret_cast<const uint4*>(p0 + C);
        const uint4 cq = *reinterpret_cast<const uint4*>(p0 + (long)W * C), d = *reinterpret_cast<const uint4*>(p0 + (long)W * C + C);
        auto mx = [](uint32_t u, uint32_t v) {
            return pack_bf16x2(fmaxf(bf16_lo(u), bf16_lo(v)), fmaxf(bf16_hi(u), bf16_hi(v)));
        };
        uint4 o;
        o.x = mx(mx(a.x, bq.x), mx(cq.x, d.x)), o.y = mx(mx(a.y, bq.y), mx(cq.y, d.y));
        o.z = mx(mx(a.z, bq.z), mx(cq.z, d.z)), o.w = mx(mx(a.w, bq.w), mx(cq.w, d.w));
        *reinterpret_cast<uint4*>(y + pix * C + c) = o;
    }
}

// dz[b,h,w,c] = (gtap[b,h,w,c] + (y[b,h,w,c] is the FIRST max of its 2x2 window ? dpool[b,h/2,w/2,c] : 0)) * (y > 0)
// One thread handles one 2x2 window x 8 channels.
__global__ void pool_relu_bwd_kernel(const __nv_bfloat16* __restrict__ y, const __nv_bfloat16* __restrict__ dpool,
                                     const __nv_bfloat16* __restrict__ gtap, __nv_bfloat16* __restrict__ dz, int B, int H,
                                     int W, int C) {
    const int Ho = H / 2, Wo = W / 2, C8 = C / 8;
    const long total = (long)B * Ho * Wo * C8;
    for (long t = blockIdx.x * (long)blockDim.x + threadIdx.x; t < total; t += (long)gridDim.x * blockDim.x) {
        const int c = (int)(t % C8) * 8;
        const long pix = t / C8;
        const int wo = (int)(pix % Wo), ho = (int)((pix / Wo) % Ho);
        const long b = pix / ((long)Wo * Ho);
        const long base = ((b * H + 2 * ho) * W + 2 * wo) * C + c;
        const long offs[4] = {0, C, (long)W * C, (long)W * C + C};
        float yv[4][8], gv[4][8], dp[8];
        {
            const uint4 q = *reinterpret_cast<const uint4*>(dpool + pix * C + c);
            const uint32_t w4[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
            for (int i = 0; i < 4; ++i) dp[2 * i] = bf16_lo(w4[i]), dp[2 * i + 1] = bf16_hi(w4[i]);
        }
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const uint4 q = *reinterpret_cast<const uint4*>(y + base + offs[k]);
            const uint32_t w4[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
            for (int i = 0; i < 4; ++i) yv[k][2 * i] = bf16_lo(w4[i]), yv[k][2 * i + 1] = bf16_hi(w4[i]);
            if (gtap) {
                const uint4 g = *reinterpret_cast<const uint4*>(gtap + base + offs[k]);
                const uint32_t g4[4] = {g.x, g.y, g.z, g.w};
#pragma unroll
                for (int i = 0; i < 4; ++i) gv[k][2 * i] = bf16_lo(g4[i]), gv[k][2 * i + 1] = bf16_hi(g4[i]);
            } else {
#pragma unroll
                for (int i = 0; i < 8; ++i) gv[k][i] = 0.f;
            }
        }
        float out[4][8];
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            int arg = 0;
            float m = yv[0][i];
#pragma unroll
            for (int k = 1; k < 4; ++k)
                if (yv[k][i] > m) m = yv[k][i], arg = k;
#pragma unroll
            for (int k = 0; k < 4; ++k) out[k][i] = (yv[k][i] > 0.f) ? gv[k][i] + (k == arg ? dp[i] : 0.f) : 0.f;
        }
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            uint4 o;
            o.x = pack_bf16x2(out[k][0], out[k][1]), o.y = pack_bf16x2(out[k][2], out[k][3]);
            o.z = pack_bf16x2(out[k][4], out[k][5]), o.w = pack_bf16x2(out[k][6], out[k][7]);
            *reinterpret_cast<uint4*>(dz + base + offs[k]) = o;
        }
    }
}

// LPP lanes per pixel, each lane owns V groups of 8 consecutive channels (16-byte loads): C = 8 * LPP * V.
// f0 (reconstruction) / f1 (target) [P][C] bf16, lin weights w[C] fp32.
//   d = Σ_c w_c (n0_c − n1_c)^2,  n = f / (||f|| + eps)      loss_acc += coef * Σ_pixels d
//   g0[P][C] = coef * d d/d f0, masked by (f0 > 0) (the tap is a ReLU output)
// (one warp per pixel left 4-byte loads and 20 full-warp shuffles per pixel at C = 64: 18 % of the HBM roofline)
template <int LPP>
__device__ __forceinline__ float group_sum(float v) {
#pragma unroll
    for (int o = LPP / 2; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ void unpack8(const uint4& u, float (&f)[8]) {
    f[0] = bf16_lo(u.x), f[1] = bf16_hi(u.x), f[2] = bf16_lo(u.y), f[3] = bf16_hi(u.y);
    f[4] = bf16_lo(u.z), f[5] = bf16_hi(u.z), f[6] = bf16_lo(u.w), f[7] = bf16_hi(u.w);
}
template <int LPP, int V>
__global__ void __launch_bounds__(256) lpips_tap_kernel(const __nv_bfloat16* __restrict__ f0, const __nv_bfloat16* __restrict__ f1,
                                                        const float* __restrict__ w, __nv_bfloat16* __restrict__ g0, long P,
                                                        float coef, float* __restrict__ loss_acc) {
    constexpr int C = 8 * LPP * V;
    constexpr int PPW = 32 / LPP;  // pixels per warp
    const long warp = (blockIdx.x * (long)blockDim.x + threadIdx.x) >> 5;
    const long nwarps = ((long)gridDim.x * blockDim.x) >> 5;
    const int lane = threadIdx.x & 31;
    const int sub = lane / LPP, li = lane % LPP;
    float wv[V][8];
#pragma unroll
    for (int v = 0; v < V; ++v) {
        const float4 wa = __ldg(reinterpret_cast<const float4*>(w + (v * LPP + li) * 8));
        const float4 wb = __ldg(reinterpret_cast<const float4*>(w + (v * LPP + li) * 8 + 4));
        wv[v][0] = wa.x, wv[v][1] = wa.y, wv[v][2] = wa.z, wv[v][3] = wa.w;
        wv[v][4] = wb.x, wv[v][5] = wb.y, wv[v][6] = wb.z, wv[v][7] = wb.w;
    }
    float local = 0.f;
    for (long base = warp * PPW; base < P; base += nwarps * PPW) {  // warp-uniform trip count
        const long pix = base + sub;
        const bool ok = pix < P;
        float a[V][8], bq[V][8];
        float s0 = 0.f, s1 = 0.f;
#pragma unroll
        for (int v = 0; v < V; ++v) {
            const long off = pix * C + (v * LPP + li) * 8;
            const uint4 u = ok ? *reinterpret_cast<const uint4*>(f0 + off) : make_uint4(0, 0, 0, 0);
            const uint4 t = ok ? *reinterpret_cast<const uint4*>(f1 + off) : make_uint4(0, 0, 0, 0);
            unpack8(u, a[v]);
            unpack8(t, bq[v]);
#pragma unroll
            for (int k = 0; k < 8; ++k) s0 += a[v][k] * a[v][k], s1 += bq[v][k] * bq[v][k];
        }
        s0 = group_sum<LPP>(s0), s1 = group_sum<LPP>(s1);
        const float r0 = sqrtf(s0), r1 = sqrtf(s1);
        const float i0 = 1.f / (r0 + 1e-10f), i1 = 1.f / (r1 + 1e-10f);
        float d = 0.f, dot = 0.f;
        float gn[V][8];
#pragma unroll
        for (int v = 0; v < V; ++v)
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                const float diff = a[v][k] * i0 - bq[v][k] * i1;
                d += wv[v][k] * diff * diff;
                gn[v][k] = 2.f * coef * wv[v][k] * diff;  // d/d n0
                dot += gn[v][k] * a[v][k];
            }
        d = group_sum<LPP>(d), dot = group_sum<LPP>(dot);
        if (li == 0 && ok) local += d;
        // g_f = gn/(r+eps) − f (gn·f) / (r (r+eps)^2)
        const float k2 = dot * i0 * i0 / fmaxf(r0, 1e-20f);
        if (ok) {
#pragma unroll
            for (int v = 0; v < V; ++v) {
                float g[8];
#pragma unroll
                for (int k = 0; k < 8; ++k) g[k] = a[v][k] > 0.f ? gn[v][k] * i0 - a[v][k] * k2 : 0.f;
                uint4 o;
                o.x = pack_bf16x2(g[0], g[1]), o.y = pack_bf16x2(g[2], g[3]);
                o.z = pack_bf16x2(g[4], g[5]), o.w = pack_bf16x2(g[6], g[7]);
                *reinterpret_cast<uint4*>(g0 + pix * C + (v * LPP + li) * 8) = o;
            }
        }
    }
    local = warp_sum(local);
    if (lane == 0 && local != 0.f) atomicAdd(loss_acc, coef * local);
}

// dcol bf16 [B*H*W][32] (k = tap*3 + c) -> dimg fp32 NCHW [B][3][H][W]: gather the 9 taps, divide by the scale
__global__ void lpips_img_grad_kernel(const __nv_bfloat16* __restrict__ dcol, float* __restrict__ dimg, int B, int H, int W) {
    const long P = (long)B * H * W;
    for (long pix = blockIdx.x * (long)blockDim.x + threadIdx.x; pix < P; pix += (long)gridDim.x * blockDim.x) {
        const int w = (int)(pix % W), h = (int)((pix / W) % H);
        const long b = pix / ((long)W * H);
        float acc[3] = {0.f, 0.f, 0.f};
#pragma unroll
        for (int tap = 0; tap < 9; ++tap) {
            // output pixel (h', w') used input (h' + dy - 1, w' + dx - 1) with this tap  =>  h' = h - dy + 1
            const int hh = h - (tap / 3) + 1, ww = w - (tap % 3) + 1;
            if (hh >= 0 && hh < H && ww >= 0 && ww < W) {
                const __nv_bfloat16* q = dcol + ((b * H + hh) * W + ww) * 32 + tap * 3;
                acc[0] += __bfloat162float(q[0]), acc[1] += __bfloat162float(q[1]), acc[2] += __bfloat162float(q[2]);
            }
        }
#pragma unroll
        for (int c = 0; c < 3; ++c) dimg[((b * 3 + c) * H + h) * W + w] = acc[c] / LP_SCALE[c];
    }
}

// ---------------------------------------------------------------- fp32-accurate metric forward (bf16x3 operands)
// img fp32 NCHW [N][3][H][W], already through the ScalingLayer -> out bf16 [N*H*W][96] = [hi|hi|lo] of the 3x3 im2col
// (k = tap*3 + c, 27 values padded to 32): the A operand of conv1_1 against [hi|lo|hi] weights (K = 96).
__global__ void lpips_prep3_kernel(const float* __restrict__ img, __nv_bfloat16* __restrict__ out, int N, int H, int W) {
    const long P = (long)N * H * W;
    for (long pix = blockIdx.x * (long)blockDim.x + threadIdx.x; pix < P; pix += (long)gridDim.x * blockDim.x) {
        const int w = (int)(pix % W), h = (int)((pix / W) % H);
        const long b = pix / ((long)W * H);
        float vals[32];
#pragma unroll
        for (int tap = 0; tap < 9; ++tap) {
            const int hh = h + tap / 3 - 1, ww = w + tap % 3 - 1;
            const bool in = hh >= 0 && hh < H && ww >= 0 && ww < W;
#pragma unroll
            for (int c = 0; c < 3; ++c) vals[tap * 3 + c] = in ? __ldg(img + ((b * 3 + c) * H + hh) * W + ww) : 0.f;
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
        uint4* o = reinterpret_cast<uint4*>(out + pix * 96);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            o[i] = make_uint4(hi[4 * i], hi[4 * i + 1], hi[4 * i + 2], hi[4 * i + 3]);
            o[4 + i] = o[i];
            o[8 + i] = make_uint4(lo[4 * i], lo[4 * i + 1], lo[4 * i + 2], lo[4 * i + 3]);
        }
    }
}

// nn.MaxPool2d(2,2) on fp32 NHWC, 4 channels per thread
__global__ void maxpool2_f32_kernel(const float* __restrict__ x, float* __restrict__ y, int B, int H, int W, int C) {
    const int Ho = H / 2, Wo = W / 2, C4 = C / 4;
    const long total = (long)B * Ho * Wo * C4;
    for (long t = blockIdx.x * (long)blockDim.x + threadIdx.x; t < total; t += (long)gridDim.x * blockDim.x) {
        const int c = (int)(t % C4) * 4;
        const long pix = t / C4;
        const int wo = (int)(pix % Wo), ho = (int)((pix / Wo) % Ho);
        const long b = pix / ((long)Wo * Ho);
        const float* p0 = x + ((b * H + 2 * ho) * W + 2 * wo) * C + c;
        const float4 a = __ldg(reinterpret_cast<const float4*>(p0)), q = __ldg(reinterpret_cast<const float4*>(p0 + C));
        const float4 r = __ldg(reinterpret_cast<const float4*>(p0 + (long)W * C));
        const float4 s = __ldg(reinterpret_cast<const float4*>(p0 + (long)W * C + C));
        float4 o;
        o.x = fmaxf(fmaxf(a.x, q.x), fmaxf(r.x, s.x)), o.y = fmaxf(fmaxf(a.y, q.y), fmaxf(r.y, s.y));
        o.z = fmaxf(fmaxf(a.z, q.z), fmaxf(r.z, s.z)), o.w = fmaxf(fmaxf(a.w, q.w), fmaxf(r.w, s.w));
        *reinterpret_cast<float4*>(y + pix * C + c) = o;
    }
}

// Forward-only LPIPS tap on fp32 NHWC features f [2n][HW][C] with the pairs interleaved (image 2i = reference,
// 2i + 1 = reconstruction): part[i*ldp + col0 + s] = (1/HW) Σ_{pixels of slice s} Σ_c w_c (f0_c/(‖f0‖+eps) − f1_c/(‖f1‖+eps))².
// grid (slices, n), one warp per pixel in a fixed assignment, fp64 block sum: no atomics.
template <int CPL>  // channels per lane (C = 32 * CPL)
__global__ void __launch_bounds__(256) lpips_tap_metric_kernel(const float* __restrict__ f, const float* __restrict__ w, int HW,
                                                               double* __restrict__ part, int ldp, int col0) {
    constexpr int C = 32 * CPL;
    __shared__ double sh[32];
    const int i = blockIdx.y, s = blockIdx.x, lane = threadIdx.x & 31;
    const int warp = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), nwarps = gridDim.x * (blockDim.x >> 5);
    const float* f0 = f + (long)(2 * i) * HW * C;
    const float* f1 = f0 + (long)HW * C;
    float wv[CPL];
#pragma unroll
    for (int k = 0; k < CPL; ++k) wv[k] = __ldg(w + k * 32 + lane);
    double local = 0.0;
    for (int p = warp; p < HW; p += nwarps) {
        float a[CPL], bq[CPL], s0 = 0.f, s1 = 0.f;
#pragma unroll
        for (int k = 0; k < CPL; ++k) {
            a[k] = __ldg(f0 + (long)p * C + k * 32 + lane), bq[k] = __ldg(f1 + (long)p * C + k * 32 + lane);
            s0 = fmaf(a[k], a[k], s0), s1 = fmaf(bq[k], bq[k], s1);
        }
        s0 = warp_sum(s0), s1 = warp_sum(s1);
        const float n0 = sqrtf(s0) + 1e-10f, n1 = sqrtf(s1) + 1e-10f;
        float d = 0.f;
#pragma unroll
        for (int k = 0; k < CPL; ++k) {
            const float diff = __fdiv_rn(a[k], n0) - __fdiv_rn(bq[k], n1);
            d = fmaf(wv[k], diff * diff, d);
        }
        local += (double)warp_sum(d);  // identical in every lane; lane 0's copy is summed below
    }
    const double tot = block_sum_f64(lane == 0 ? local : 0.0, sh);
    if (threadIdx.x == 0) part[(long)i * ldp + col0 + s] = tot / HW;
}

static inline int gridn(long n, int block) {
    long g = (n + block - 1) / block;
    long cap = (long)num_sms() * 16;
    return (int)(g < 1 ? 1 : (g < cap ? g : cap));
}

}  // namespace vtp

using namespace vtp;

extern "C" int vtp_lpips_prep(const void* img, int img_dtype, void* out_bf16, int B, int H, int W, vtp_stream_t st) {
    VTP_CHECK_ARG(img && out_bf16 && B > 0 && H > 0 && W > 0, "lpips_prep: bad args");
    const long P = (long)B * H * W;
    if (img_dtype == VTP_F32)
        lpips_prep_kernel<float><<<gridn(P, 128), 128, 0, (cudaStream_t)st>>>((const float*)img, (__nv_bfloat16*)out_bf16, B, H, W);
    else
        lpips_prep_kernel<__nv_bfloat16>
            <<<gridn(P, 128), 128, 0, (cudaStream_t)st>>>((const __nv_bfloat16*)img, (__nv_bfloat16*)out_bf16, B, H, W);
    VTP_LAUNCH_CHECK();
    return VTP_OK;
}

extern "C" int vtp_maxpool2_fwd(const void* x, void* y, int B, int H, int W, int C, vtp_stream_t st) {
    VTP_CHECK_ARG(x && y && B > 0 && H % 2 == 0 && W % 2 == 0 && C % 8 == 0, "maxpool2_fwd: bad args");
    const long total = (long)B * (H / 2) * (W / 2) * (C / 8);
    maxpool2_fwd_kernel<<<gridn(total, 256), 256, 0, (cudaStream_t)st>>>((const __nv_bfloat16*)x, (__nv_bfloat16*)y, B, H, W, C);
    VTP_LAUNCH_CHECK();
    return VTP_OK;
}

extern "C" int vtp_pool_relu_bwd(const void* y, const void* dpool, const void* gtap, void* dz, int B, int H, int W, int C,
                                 vtp_stream_t st) {
    VTP_CHECK_ARG(y && dpool && dz && B > 0 && H % 2 == 0 && W % 2 == 0 && C % 8 == 0, "pool_relu_bwd: bad args");
    const long total = (long)B * (H / 2) * (W / 2) * (C / 8);
    pool_relu_bwd_kernel<<<gridn(total, 128), 128, 0, (cudaStream_t)st>>>((const __nv_bfloat16*)y, (const __nv_bfloat16*)dpool,
                                                                          (const __nv_bfloat16*)gtap, (__nv_bfloat16*)dz, B, H, W, C);
    VTP_LAUNCH_CHECK();
    return VTP_OK;
}

extern "C" int vtp_lpips_tap(const void* f0, const void* f1, const float* w, void* g0, long P, int C, float coef,
                             float* loss_acc, vtp_stream_t st) {
    VTP_CHECK_ARG(f0 && f1 && w && g0 && loss_acc && P > 0 && C % 64 == 0 && C <= 512, "lpips_tap: bad args (C %% 64, C <= 512)");
    const __nv_bfloat16 *a0 = (const __nv_bfloat16*)f0, *a1 = (const __nv_bfloat16*)f1;
    __nv_bfloat16* g = (__nv_bfloat16*)g0;
    cudaStream_t stream = (cudaStream_t)st;
    switch (C) {
        case 64: lpips_tap_kernel<8, 1><<<gridn(P * 8, 256), 256, 0, stream>>>(a0, a1, w, g, P, coef, loss_acc); break;
        case 128: lpips_tap_kernel<16, 1><<<gridn(P * 16, 256), 256, 0, stream>>>(a0, a1, w, g, P, coef, loss_acc); break;
        case 256: lpips_tap_kernel<32, 1><<<gridn(P * 32, 256), 256, 0, stream>>>(a0, a1, w, g, P, coef, loss_acc); break;
        case 512: lpips_tap_kernel<32, 2><<<gridn(P * 32, 256), 256, 0, stream>>>(a0, a1, w, g, P, coef, loss_acc); break;
        default: VTP_FAIL(VTP_ERR_ARG, "lpips_tap: C = %d not in {64, 128, 256, 512}", C);
    }
    VTP_LAUNCH_CHECK();
    return VTP_OK;
}

extern "C" int vtp_lpips_prep3(const float* img, void* out_bf16, int N, int H, int W, vtp_stream_t st) {
    VTP_CHECK_ARG(img && out_bf16 && N > 0 && H > 0 && W > 0 && ((uintptr_t)out_bf16 & 15) == 0, "lpips_prep3: bad args");
    const long P = (long)N * H * W;
    lpips_prep3_kernel<<<gridn(P, 128), 128, 0, (cudaStream_t)st>>>(img, (__nv_bfloat16*)out_bf16, N, H, W);
    VTP_LAUNCH_CHECK();
    return VTP_OK;
}

extern "C" int vtp_maxpool2_f32(const float* x, float* y, int B, int H, int W, int C, vtp_stream_t st) {
    VTP_CHECK_ARG(x && y && B > 0 && H % 2 == 0 && W % 2 == 0 && C % 4 == 0, "maxpool2_f32: bad args (even H, W; C %% 4)");
    const long total = (long)B * (H / 2) * (W / 2) * (C / 4);
    maxpool2_f32_kernel<<<gridn(total, 256), 256, 0, (cudaStream_t)st>>>(x, y, B, H, W, C);
    VTP_LAUNCH_CHECK();
    return VTP_OK;
}

extern "C" int vtp_lpips_tap_metric(const float* f, const float* w, int n, int HW, int C, double* part, int ldp, int col0,
                                    int slices, vtp_stream_t st) {
    VTP_CHECK_ARG(f && w && part && n > 0 && n <= 65535 && HW > 0 && slices > 0 && col0 >= 0 && col0 + slices <= ldp,
                  "lpips_tap_metric: bad args (col0 + slices <= ldp)");
    const dim3 grid(slices, n);
    cudaStream_t stream = (cudaStream_t)st;
    switch (C) {
        case 64: lpips_tap_metric_kernel<2><<<grid, 256, 0, stream>>>(f, w, HW, part, ldp, col0); break;
        case 128: lpips_tap_metric_kernel<4><<<grid, 256, 0, stream>>>(f, w, HW, part, ldp, col0); break;
        case 256: lpips_tap_metric_kernel<8><<<grid, 256, 0, stream>>>(f, w, HW, part, ldp, col0); break;
        case 512: lpips_tap_metric_kernel<16><<<grid, 256, 0, stream>>>(f, w, HW, part, ldp, col0); break;
        default: VTP_FAIL(VTP_ERR_ARG, "lpips_tap_metric: C = %d not in {64, 128, 256, 512}", C);
    }
    VTP_LAUNCH_CHECK();
    return VTP_OK;
}

extern "C" int vtp_lpips_img_grad(const void* dcol, float* dimg, int B, int H, int W, vtp_stream_t st) {
    VTP_CHECK_ARG(dcol && dimg && B > 0, "lpips_img_grad: bad args");
    lpips_img_grad_kernel<<<gridn((long)B * H * W, 256), 256, 0, (cudaStream_t)st>>>((const __nv_bfloat16*)dcol, dimg, B, H, W);
    VTP_LAUNCH_CHECK();
    return VTP_OK;
}
