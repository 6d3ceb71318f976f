// vtp_b200 — input side of the training step (SURVEY.md §8f rank 4; absent from the reference, which leaves multi-crop /
// mask generation / tokenisation to an un-released DINOv2-style CPU data loader): ONE kernel turns the decoded uint8 source
// images (NHWC, as a JPEG decoder / DataLoader delivers them) into every normalised fp32 NCHW crop of the step.
//
//   crop n :  source image src_idx[n], box (x0, y0, w, h) in source pixels (fractional allowed), optional horizontal flip,
//             bilinear resample to S x S with half-pixel centres (== F.interpolate(..., mode="bilinear",
//             align_corners=False, antialias=False) of the cropped region), then (v / 255 - mean[c]) / std[c].
// One thread = one output pixel (3 channels): the 4 taps x 3 bytes come from L2 (a 256 x 256 x 3 source is 192 KB), the
// store is three coalesced fp32 writes.  HBM-bound on the output: 12 B per output pixel.
//
// vtp_crop_augment adds DINOv2's photometric augmentations between the resample and the normalisation (colour jitter in a
// per-crop order, grayscale, 9-tap Gaussian blur with reflect padding, solarise; torchvision.transforms.v2.functional
// semantics on float images).  Two kernels:
//   crop_augment_stats_kernel  one CTA per crop: the grayscale mean contrast blends towards, over the image as it stands
//                              when contrast runs (resample + the jitter ops before it, recomputed from the source).
//   crop_augment_kernel        one CTA per 32 x 32 output tile: resample + colour chain for the tile and a 4-pixel
//                              reflect-indexed halo into shared memory, separable blur, solarise, normalise, store.
// Both carry pixel values in 0..255 units, the unit the resample produces, so that a crop with every stage off stores the
// very expression crop_resize_norm_kernel stores.  Every op is scale-free or scaled with it (clamp bound 255, solarise
// threshold 255 t, 255 - x).  No atomics: reductions run in a fixed order, so repeat launches are bit-identical.
#include "host.h"
#include "ptx.cuh"

namespace vtp {

// bilinear sample of output pixel (xo, oy) (xo already flipped) of box bx, in 0..255 units
__device__ __forceinline__ void sample_rgb(const uint8_t* __restrict__ img, int H, int W, float4 bx, int xo, int oy, int S,
                                           float v[3]) {
    // half-pixel centres: source coordinate of the output pixel centre, clamped like torch's bilinear kernel
    float sx = bx.x + (xo + 0.5f) * (bx.z / S) - 0.5f;
    float sy = bx.y + (oy + 0.5f) * (bx.w / S) - 0.5f;
    // torch clamps the coordinate inside the CROPPED tensor; in source coordinates that is [x0, x0 + w - 1]
    sx = fminf(fmaxf(sx, bx.x), bx.x + bx.z - 1.f);
    sy = fminf(fmaxf(sy, bx.y), bx.y + bx.w - 1.f);
    const int x0 = (int)floorf(sx), y0 = (int)floorf(sy);
    const float fx = sx - x0, fy = sy - y0;
    const int xa = min(max(x0, 0), W - 1), xb = min(max(x0 + 1, 0), W - 1);
    const int ya = min(max(y0, 0), H - 1), yb = min(max(y0 + 1, 0), H - 1);
    const uint8_t* p00 = img + ((long)ya * W + xa) * 3;
    const uint8_t* p01 = img + ((long)ya * W + xb) * 3;
    const uint8_t* p10 = img + ((long)yb * W + xa) * 3;
    const uint8_t* p11 = img + ((long)yb * W + xb) * 3;
    const float w00 = (1.f - fx) * (1.f - fy), w01 = fx * (1.f - fy), w10 = (1.f - fx) * fy, w11 = fx * fy;
#pragma unroll
    for (int c = 0; c < 3; ++c) v[c] = w00 * p00[c] + w01 * p01[c] + w10 * p10[c] + w11 * p11[c];
}

__device__ __forceinline__ float normalize(float v, float m, float is) { return (v * (1.f / 255.f) - m) * is; }

__global__ void crop_resize_norm_kernel(const uint8_t* __restrict__ src, int H, int W, const int* __restrict__ src_idx,
                                        const float* __restrict__ boxes, const uint8_t* __restrict__ flips,
                                        float* __restrict__ out, int N, int S, float m0, float m1, float m2, float is0,
                                        float is1, float is2) {
    const long per = (long)S * S, total = (long)N * per;
    for (long t = blockIdx.x * (long)blockDim.x + threadIdx.x; t < total; t += (long)gridDim.x * blockDim.x) {
        const int n = (int)(t / per), r = (int)(t - (long)n * per);
        const int oy = r / S, ox = r - oy * S;
        const float4 bx = __ldg(reinterpret_cast<const float4*>(boxes) + n);   // x0, y0, w, h
        const int xo = flips && flips[n] ? S - 1 - ox : ox;
        float v[3];
        sample_rgb(src + (long)src_idx[n] * H * W * 3, H, W, bx, xo, oy, S, v);
        float* o = out + (long)n * 3 * per + r;
        o[0] = normalize(v[0], m0, is0);
        o[per] = normalize(v[1], m1, is1);
        o[2 * per] = normalize(v[2], m2, is2);
    }
}

// ------------------------------------------------------------------------------------------------ photometric stages
// itertools.permutations(range(4)) in its order, op k of permutation p in bits 2k..2k+1 (0 brightness, 1 contrast,
// 2 saturation, 3 hue)
__constant__ uint8_t kJitterOrders[24] = {0xe4, 0xb4, 0xd8, 0x78, 0x9c, 0x6c, 0xe1, 0xb1, 0xc9, 0x39, 0x8d, 0x2d,
                                          0xd2, 0x72, 0xc6, 0x36, 0x4e, 0x1e, 0x93, 0x63, 0x87, 0x27, 0x4b, 0x1b};

__device__ __forceinline__ float clamp255(float v) { return fminf(fmaxf(v, 0.f), 255.f); }
__device__ __forceinline__ float gray(const float x[3]) { return 0.2989f * x[0] + 0.587f * x[1] + 0.114f * x[2]; }

// torchvision _rgb_to_hsv, hue + dh wrapped by a floored remainder, _hsv_to_rgb (sector = floor(6h) floored mod 6)
__device__ __forceinline__ void hue_shift(float x[3], float dh) {
    const float r = x[0], g = x[1], b = x[2];
    const float maxc = fmaxf(r, fmaxf(g, b)), minc = fminf(r, fminf(g, b));
    const bool eqc = maxc == minc;
    const float cr = maxc - minc;
    const float s = cr / (eqc ? 1.f : maxc);
    const float dv = eqc ? 1.f : cr;
    const float rc = (maxc - r) / dv, gc = (maxc - g) / dv, bc = (maxc - b) / dv;
    float h = maxc == r ? bc - gc : maxc == g ? 2.f + rc - bc : 4.f + gc - rc;   // tie rule: r first, then g
    h = fmodf(h * (1.f / 6.f) + 1.f, 1.f);
    h = fmodf(h + dh, 1.f);
    if (h < 0.f) h += 1.f;
    const float h6 = h * 6.f, fl = floorf(h6), f = h6 - fl;
    int i = (int)fl % 6;
    if (i < 0) i += 6;
    const float sxf = s * f, oms = 1.f - s;
    const float v = maxc, q = clamp255((1.f - sxf) * v), t = clamp255((sxf + oms) * v), p = clamp255(oms * v);
    switch (i) {
        case 0: x[0] = v; x[1] = t; x[2] = p; break;
        case 1: x[0] = q; x[1] = v; x[2] = p; break;
        case 2: x[0] = p; x[1] = v; x[2] = t; break;
        case 3: x[0] = p; x[1] = q; x[2] = v; break;
        case 4: x[0] = t; x[1] = p; x[2] = v; break;
        default: x[0] = v; x[1] = p; x[2] = q; break;
    }
}

// one colour-jitter op (torchvision adjust_*: _blend and a clamp after each); f = brightness, contrast, saturation, hue
__device__ __forceinline__ void jitter_op(int op, float x[3], float4 f, float cmean) {
    if (op == 0) {
#pragma unroll
        for (int c = 0; c < 3; ++c) x[c] = clamp255(f.x * x[c]);
    } else if (op == 1) {
#pragma unroll
        for (int c = 0; c < 3; ++c) x[c] = clamp255(f.y * x[c] + (1.f - f.y) * cmean);
    } else if (op == 2) {
        const float g = gray(x);
#pragma unroll
        for (int c = 0; c < 3; ++c) x[c] = clamp255(f.z * x[c] + (1.f - f.z) * g);
    } else {
        hue_shift(x, f.w);
    }
}

struct CropArgs {
    const uint8_t* src;
    int H, W, S;
    const int* src_idx;
    const float* boxes;
    const uint8_t* flips;
    const float* params;
};

constexpr int STATS_THREADS = 1024;

__global__ void __launch_bounds__(STATS_THREADS) crop_augment_stats_kernel(CropArgs a, float* __restrict__ mean_ws) {
    const int n = blockIdx.x;
    const float4 f = __ldg(reinterpret_cast<const float4*>(a.params) + 2 * n);
    const int code = (int)__ldg(a.params + 8 * n + 4);
    if (code < 0) return;                        // no jitter, so no contrast: the apply kernel never reads mean_ws[n]
    const unsigned ord = kJitterOrders[code];
    int pre = 0;
    while (((ord >> (2 * pre)) & 3u) != 1u) ++pre;   // ops before contrast
    const float4 bx = __ldg(reinterpret_cast<const float4*>(a.boxes) + n);
    const bool flip = a.flips && a.flips[n];
    const uint8_t* img = a.src + (long)a.src_idx[n] * a.H * a.W * 3;
    const int S = a.S;
    const long per = (long)S * S;
    double acc = 0.0;
    for (long t = threadIdx.x; t < per; t += STATS_THREADS) {
        const int oy = (int)(t / S), ox = (int)(t - (long)oy * S);
        float x[3];
        sample_rgb(img, a.H, a.W, bx, flip ? S - 1 - ox : ox, oy, S, x);
#pragma unroll 1
        for (int k = 0; k < pre; ++k) jitter_op((ord >> (2 * k)) & 3u, x, f, 0.f);
        acc += gray(x);
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) acc += __shfl_down_sync(0xffffffffu, acc, off);
    __shared__ double part[STATS_THREADS / 32];
    if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        double s = 0.0;
        for (int w = 0; w < STATS_THREADS / 32; ++w) s += part[w];
        mean_ws[n] = (float)(s / (double)per);
    }
}

constexpr int TILE = 32, HALO = 4, TW = TILE + 2 * HALO, APPLY_THREADS = 256;

// reflect padding (valid for p in [-4, S + 3] when S >= 5); positions further out only feed outputs past the crop's
// edge, which are never stored, and are clamped so that they stay inside the source box
__device__ __forceinline__ int reflect(int p, int S) {
    p = p < 0 ? -p : p;
    p = p >= S ? 2 * (S - 1) - p : p;
    return max(p, 0);
}

__global__ void __launch_bounds__(APPLY_THREADS) crop_augment_kernel(CropArgs a, const float* __restrict__ mean_ws,
                                                                     float* __restrict__ out, int tiles_x, float m0,
                                                                     float m1, float m2, float is0, float is1,
                                                                     float is2) {
    __shared__ float cs[3][TW][TW];    // colour-chained tile + halo
    __shared__ float hs[3][TW][TILE];  // after the horizontal blur
    __shared__ float wk[9];
    const int tiles = tiles_x * tiles_x;
    const int n = blockIdx.x / tiles, tile = blockIdx.x - n * tiles;
    const int ty0 = (tile / tiles_x) * TILE, tx0 = (tile - (tile / tiles_x) * tiles_x) * TILE;
    const int S = a.S;
    const float4 f = __ldg(reinterpret_cast<const float4*>(a.params) + 2 * n);
    const float4 g = __ldg(reinterpret_cast<const float4*>(a.params) + 2 * n + 1);
    const int code = (int)g.x;
    const unsigned ord = code >= 0 ? kJitterOrders[code] : 0u;
    const float cmean = code >= 0 ? mean_ws[n] : 0.f;
    const bool to_gray = g.y != 0.f;
    const float sigma = g.z, t255 = g.w * 255.f;
    const float4 bx = __ldg(reinterpret_cast<const float4*>(a.boxes) + n);
    const bool flip = a.flips && a.flips[n];
    const uint8_t* img = a.src + (long)a.src_idx[n] * a.H * a.W * 3;
    const long per = (long)S * S;
    float* o = out + (long)n * 3 * per;

    auto colour = [&](int oy, int ox, float x[3]) {
        sample_rgb(img, a.H, a.W, bx, flip ? S - 1 - ox : ox, oy, S, x);
        if (code >= 0) {
#pragma unroll 1
            for (int k = 0; k < 4; ++k) jitter_op((ord >> (2 * k)) & 3u, x, f, cmean);
        }
        if (to_gray) x[0] = x[1] = x[2] = gray(x);
    };
    auto store = [&](int oy, int ox, const float x[3]) {
        const long r = (long)oy * S + ox;
        float v0 = x[0] >= t255 ? 255.f - x[0] : x[0];
        float v1 = x[1] >= t255 ? 255.f - x[1] : x[1];
        float v2 = x[2] >= t255 ? 255.f - x[2] : x[2];
        o[r] = normalize(v0, m0, is0);
        o[per + r] = normalize(v1, m1, is1);
        o[2 * per + r] = normalize(v2, m2, is2);
    };

    if (!(sigma > 0.f)) {
        for (int i = threadIdx.x; i < TILE * TILE; i += APPLY_THREADS) {
            const int oy = ty0 + i / TILE, ox = tx0 + i % TILE;
            if (oy >= S || ox >= S) continue;
            float x[3];
            colour(oy, ox, x);
            store(oy, ox, x);
        }
        return;
    }
    if (threadIdx.x < 9) {   // exp(-x^2 / 2 sigma^2), x = -4..4, normalised; each thread sums all nine in the same order
        float s = 0.f;
#pragma unroll
        for (int j = -HALO; j <= HALO; ++j) s += expf(-0.5f * (j / sigma) * (j / sigma));
        const float j = (float)((int)threadIdx.x - HALO);
        wk[threadIdx.x] = expf(-0.5f * (j / sigma) * (j / sigma)) / s;
    }
    for (int i = threadIdx.x; i < TW * TW; i += APPLY_THREADS) {
        const int ly = i / TW, lx = i - ly * TW;
        float x[3];
        colour(reflect(ty0 + ly - HALO, S), reflect(tx0 + lx - HALO, S), x);
#pragma unroll
        for (int c = 0; c < 3; ++c) cs[c][ly][lx] = x[c];
    }
    __syncthreads();
    for (int i = threadIdx.x; i < TW * TILE; i += APPLY_THREADS) {
        const int r = i / TILE, cx = i % TILE;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            float s = 0.f;
#pragma unroll
            for (int k = 0; k < 9; ++k) s += wk[k] * cs[c][r][cx + k];
            hs[c][r][cx] = s;
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < TILE * TILE; i += APPLY_THREADS) {
        const int y = i / TILE, x = i % TILE, oy = ty0 + y, ox = tx0 + x;
        if (oy >= S || ox >= S) continue;
        float v[3];
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            float s = 0.f;
#pragma unroll
            for (int k = 0; k < 9; ++k) s += wk[k] * hs[c][y + k][x];
            v[c] = s;
        }
        store(oy, ox, v);
    }
}

}  // namespace vtp

extern "C" int vtp_crop_resize_norm(const uint8_t* src_nhwc, int B, int H, int W, const int* src_idx, const float* boxes_xywh,
                                    const uint8_t* flips, float* out_nchw, int N, int S, const float* mean3,
                                    const float* std3, vtp_stream_t st) {
    VTP_CHECK_ARG(src_nhwc && src_idx && boxes_xywh && out_nchw && mean3 && std3 && B > 0 && H > 0 && W > 0 && N > 0 && S > 0,
                  "crop_resize_norm: bad args");
    VTP_CHECK_ARG((reinterpret_cast<uintptr_t>(boxes_xywh) & 15) == 0, "crop_resize_norm: boxes must be 16B aligned");
    const long total = (long)N * S * S;
    long g = (total + 255) / 256;
    const long cap = (long)vtp::num_sms() * 16;
    vtp::crop_resize_norm_kernel<<<(int)(g < cap ? g : cap), 256, 0, (cudaStream_t)st>>>(
        src_nhwc, H, W, src_idx, boxes_xywh, flips, out_nchw, N, S, mean3[0], mean3[1], mean3[2], 1.f / std3[0], 1.f / std3[1],
        1.f / std3[2]);
    VTP_LAUNCH_CHECK();
    return VTP_OK;
}

extern "C" int vtp_crop_augment(const uint8_t* src_nhwc, int B, int H, int W, const int* src_idx, const float* boxes_xywh,
                                const uint8_t* flips, const float* params, float* mean_ws, float* out_nchw, int N, int S,
                                const float* mean3, const float* std3, vtp_stream_t st) {
    VTP_CHECK_ARG(src_nhwc && src_idx && boxes_xywh && params && mean_ws && out_nchw && mean3 && std3 && B > 0 && H > 0 &&
                      W > 0 && N > 0,
                  "crop_augment: bad args");
    VTP_CHECK_ARG(S >= 5, "crop_augment: S = %d, the 9-tap blur's reflect padding needs S >= 5", S);
    VTP_CHECK_ARG((reinterpret_cast<uintptr_t>(boxes_xywh) & 15) == 0, "crop_augment: boxes must be 16B aligned");
    VTP_CHECK_ARG((reinterpret_cast<uintptr_t>(params) & 15) == 0, "crop_augment: params must be 16B aligned");
    const int tiles_x = (S + vtp::TILE - 1) / vtp::TILE;
    const long ctas = (long)N * tiles_x * tiles_x;
    VTP_CHECK_ARG(ctas < (1L << 31), "crop_augment: %ld tiles exceed one launch", ctas);
    const vtp::CropArgs a{src_nhwc, H, W, S, src_idx, boxes_xywh, flips, params};
    vtp::crop_augment_stats_kernel<<<N, vtp::STATS_THREADS, 0, (cudaStream_t)st>>>(a, mean_ws);
    VTP_LAUNCH_CHECK();
    vtp::crop_augment_kernel<<<(int)ctas, vtp::APPLY_THREADS, 0, (cudaStream_t)st>>>(
        a, mean_ws, out_nchw, tiles_x, mean3[0], mean3[1], mean3[2], 1.f / std3[0], 1.f / std3[1], 1.f / std3[2]);
    VTP_LAUNCH_CHECK();
    return VTP_OK;
}
