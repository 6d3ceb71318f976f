// vtp_b200 — reconstruction metrics of tools/test_reconstruction_hf.py (PSNR :49-62,395-397, torchmetrics SSIM :392,
// the uint8 PNG pixels :401-402) over one batch of (input, reconstruction) pairs, without a host read:
//   recon_pixels    one pass over both images: denormalise + clamp in registers; uint8 NHWC copies, the LPIPS network
//                   input (x·2−1, ScalingLayer) and per-(image, band) fp64 sums of the squared error
//   recon_ssim      11x11 Gaussian SSIM over the windows wholly inside the image, from shared-memory tiles with a
//                   10-pixel halo; per-(image, tile) fp64 partial sums
//   recon_finalise  per-image PSNR / SSIM / LPIPS from the partials in a fixed order, batch means into fp64
//                   accumulators
// No atomics anywhere: repeated runs are bit-identical.
#include "host.h"
#include "ptx.cuh"

namespace vtp {

constexpr int SSIM_TILE = 32;                 // valid-window outputs per tile side
constexpr int SSIM_IN = SSIM_TILE + 10;       // input rows / columns per tile (10-pixel halo)
constexpr float SSIM_C1 = 0.01f * 0.01f, SSIM_C2 = 0.03f * 0.03f;

__constant__ float RM_SHIFT[3] = {-0.030f, -0.088f, -0.188f};
__constant__ float RM_SCALE[3] = {0.458f, 0.448f, 0.450f};

// torchvision Normalize(-m/s, 1/s) = (v − sub) / div in fp32 (no contraction), then torch.clamp(·, 0, 1) (NaN kept)
__device__ __forceinline__ float denorm_clamp(float v, float sub, float div) {
    const float t = __fdiv_rn(__fsub_rn(v, sub), div);
    return t != t ? t : fminf(fmaxf(t, 0.f), 1.f);
}
__device__ __forceinline__ float ld_any(const float* p) { return __ldg(p); }
__device__ __forceinline__ float ld_any(const __nv_bfloat16* p) { return __bfloat162float(*p); }

// grid (bands, B), 256 threads; band j covers rows [j*rows, (j+1)*rows).
template <typename TR>
__global__ void __launch_bounds__(256) recon_pixels_kernel(const float* __restrict__ x, const TR* __restrict__ rec, int H, int W,
                                                           const float* __restrict__ sub3, const float* __restrict__ div3,
                                                           int rows, uint8_t* __restrict__ u8_ref, uint8_t* __restrict__ u8_rec,
                                                           float* __restrict__ lp, double* __restrict__ sse_part) {
    __shared__ double sh[32];
    const int b = blockIdx.y, band = blockIdx.x;
    const long HW = (long)H * W;
    const int r0 = band * rows, r1 = min(H, r0 + rows);
    const float sub[3] = {sub3[0], sub3[1], sub3[2]}, div[3] = {div3[0], div3[1], div3[2]};
    double sse = 0.0;
    for (long q = (long)r0 * W + threadIdx.x; q < (long)r1 * W; q += blockDim.x) {
        unsigned uo[3], ur[3];
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const long i = ((long)b * 3 + c) * HW + q;
            const float o = denorm_clamp(__ldg(x + i), sub[c], div[c]);
            const float r = denorm_clamp(ld_any(rec + i), sub[c], div[c]);
            const float o255 = __fmul_rn(o, 255.f), r255 = __fmul_rn(r, 255.f);
            const float d = __fsub_rn(o255, r255);
            sse += (double)d * (double)d;
            uo[c] = o255 == o255 ? (unsigned)o255 : 0u;  // astype(uint8) truncates; NaN -> 0 as vtp_image_to_u8
            ur[c] = r255 == r255 ? (unsigned)r255 : 0u;
            if (lp) {  // LPIPS input (test_reconstruction_hf.py:381-382) through the ScalingLayer (lpips.py:113-114)
                lp[(((long)b * 2 + 0) * 3 + c) * HW + q] =
                    __fdiv_rn(__fsub_rn(__fsub_rn(__fmul_rn(o, 2.f), 1.f), RM_SHIFT[c]), RM_SCALE[c]);
                lp[(((long)b * 2 + 1) * 3 + c) * HW + q] =
                    __fdiv_rn(__fsub_rn(__fsub_rn(__fmul_rn(r, 2.f), 1.f), RM_SHIFT[c]), RM_SCALE[c]);
            }
        }
        if (u8_ref) {
            uint8_t* po = u8_ref + ((long)b * HW + q) * 3;
            uint8_t* pr = u8_rec + ((long)b * HW + q) * 3;
#pragma unroll
            for (int c = 0; c < 3; ++c) po[c] = (uint8_t)uo[c], pr[c] = (uint8_t)ur[c];
        }
    }
    sse = block_sum_f64(sse, sh);
    if (threadIdx.x == 0) sse_part[(long)b * gridDim.x + band] = sse;
}

// grid (tiles_x, tiles_y, B), 256 threads.  Output (valid-window) position (oy, ox) is the window whose top-left input
// pixel is (oy, ox), i.e. torchmetrics' map pixel (oy + 5, ox + 5) after the reflect pad and the 5-pixel crop.
template <typename TR>
__global__ void __launch_bounds__(256) recon_ssim_kernel(const float* __restrict__ x, const TR* __restrict__ rec, int H, int W,
                                                         const float* __restrict__ sub3, const float* __restrict__ div3,
                                                         double* __restrict__ part) {
    __shared__ float sx[SSIM_IN][SSIM_IN + 1], sy[SSIM_IN][SSIM_IN + 1];
    __shared__ float hm[5][SSIM_IN][SSIM_TILE + 1];
    __shared__ float g[11];
    __shared__ double sh[32];
    const int b = blockIdx.z, oy0 = blockIdx.y * SSIM_TILE, ox0 = blockIdx.x * SSIM_TILE;
    const int Ho = H - 10, Wo = W - 10;
    const long HW = (long)H * W;
    if (threadIdx.x == 0) {  // torchmetrics _gaussian: exp(−(d/σ)²/2), d = −5..5, σ = 1.5, normalised (fp32)
        float t[11], s = 0.f;
        for (int k = 0; k < 11; ++k) {
            const float d = __fdiv_rn((float)(k - 5), 1.5f);
            t[k] = expf(-__fmul_rn(d, d) / 2.f);
            s += t[k];
        }
        for (int k = 0; k < 11; ++k) g[k] = t[k] / s;
    }
    double acc = 0.0;
    for (int c = 0; c < 3; ++c) {
        const float sub = sub3[c], div = div3[c];
        __syncthreads();
        for (int i = threadIdx.x; i < SSIM_IN * SSIM_IN; i += blockDim.x) {
            const int r = i / SSIM_IN, col = i % SSIM_IN, yy = oy0 + r, xx = ox0 + col;
            float a = 0.f, bb = 0.f;
            if (yy < H && xx < W) {
                const long off = ((long)b * 3 + c) * HW + (long)yy * W + xx;
                a = denorm_clamp(__ldg(x + off), sub, div);
                bb = denorm_clamp(ld_any(rec + off), sub, div);
            }
            sx[r][col] = a, sy[r][col] = bb;
        }
        __syncthreads();
        for (int i = threadIdx.x; i < SSIM_IN * SSIM_TILE; i += blockDim.x) {  // horizontal 11-tap pass
            const int r = i / SSIM_TILE, col = i % SSIM_TILE;
            float m0 = 0.f, m1 = 0.f, m2 = 0.f, m3 = 0.f, m4 = 0.f;
#pragma unroll
            for (int k = 0; k < 11; ++k) {
                const float a = sx[r][col + k], bb = sy[r][col + k], w = g[k];
                m0 = fmaf(w, a, m0), m1 = fmaf(w, bb, m1);
                m2 = fmaf(w, a * a, m2), m3 = fmaf(w, bb * bb, m3), m4 = fmaf(w, a * bb, m4);
            }
            hm[0][r][col] = m0, hm[1][r][col] = m1, hm[2][r][col] = m2, hm[3][r][col] = m3, hm[4][r][col] = m4;
        }
        __syncthreads();
        for (int i = threadIdx.x; i < SSIM_TILE * SSIM_TILE; i += blockDim.x) {  // vertical pass + SSIM map
            const int r = i / SSIM_TILE, col = i % SSIM_TILE;
            if (oy0 + r >= Ho || ox0 + col >= Wo) continue;
            float mu_x = 0.f, mu_y = 0.f, exx = 0.f, eyy = 0.f, exy = 0.f;
#pragma unroll
            for (int k = 0; k < 11; ++k) {
                const float w = g[k];
                mu_x = fmaf(w, hm[0][r + k][col], mu_x), mu_y = fmaf(w, hm[1][r + k][col], mu_y);
                exx = fmaf(w, hm[2][r + k][col], exx), eyy = fmaf(w, hm[3][r + k][col], eyy);
                exy = fmaf(w, hm[4][r + k][col], exy);
            }
            // torchmetrics functional/image/ssim.py _ssim_update, in its order of operations
            const float mxx = mu_x * mu_x, myy = mu_y * mu_y, mxy = mu_x * mu_y;
            const float vx = fmaxf(exx - mxx, 0.f), vy = fmaxf(eyy - myy, 0.f), cxy = exy - mxy;
            const float upper = 2.f * cxy + SSIM_C2, lower = (vx + vy) + SSIM_C2;
            acc += (double)(((2.f * mxy + SSIM_C1) * upper) / ((mxx + myy + SSIM_C1) * lower));
        }
    }
    acc = block_sum_f64(acc, sh);
    if (threadIdx.x == 0) part[(long)b * gridDim.x * gridDim.y + (long)blockIdx.y * gridDim.x + blockIdx.x] = acc;
}

// One CTA.  acc: [0] Σ PSNR over images, [1] images, [2] Σ batch-mean SSIM, [3] Σ batch-mean LPIPS, [4] batches.
__global__ void recon_finalise_kernel(const double* __restrict__ sse_part, int nbands, const double* __restrict__ ssim_part,
                                      int ntiles, const double* __restrict__ lp_part, int nlp, int B, double npix,
                                      double nwin, double* __restrict__ psnr, float* __restrict__ ssim,
                                      float* __restrict__ lpips, double* __restrict__ acc) {
    for (int b = threadIdx.x; b < B; b += blockDim.x) {
        double s = 0.0;
        for (int j = 0; j < nbands; ++j) s += sse_part[(long)b * nbands + j];
        const double mse = s / npix;  // mean over the 3·H·W values of ((o − r)·255)²
        psnr[b] = mse == 0.0 ? __longlong_as_double(0x7ff0000000000000LL) : 20.0 * log10(255.0 / sqrt(mse));
        s = 0.0;
        for (int j = 0; j < ntiles; ++j) s += ssim_part[(long)b * ntiles + j];
        ssim[b] = (float)(s / nwin);
        if (lp_part) {
            s = 0.0;
            for (int j = 0; j < nlp; ++j) s += lp_part[(long)b * nlp + j];
            lpips[b] = (float)s;
        }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        double sp = 0.0, ss = 0.0, sl = 0.0;
        for (int b = 0; b < B; ++b) {
            sp += psnr[b];
            ss += (double)ssim[b];
            if (lp_part) sl += (double)lpips[b];
        }
        acc[0] += sp;
        acc[1] += B;
        acc[2] += ss / B;
        if (lp_part) acc[3] += sl / B;
        acc[4] += 1.0;
    }
}

}  // namespace vtp

using namespace vtp;

extern "C" int vtp_recon_pixels(const float* x, const void* rec, int rec_dtype, int B, int H, int W, const float* sub3,
                                const float* div3, uint8_t* u8_ref, uint8_t* u8_rec, float* lp, double* sse_part,
                                int nbands, vtp_stream_t st) {
    VTP_CHECK_ARG(x && rec && sub3 && div3 && sse_part && B > 0 && B <= 65535 && H > 0 && W > 0 && nbands > 0 &&
                      nbands <= 65535 && (rec_dtype == VTP_F32 || rec_dtype == VTP_BF16) && (!u8_ref == !u8_rec),
                  "recon_pixels: bad args (0 < B, nbands <= 65535; u8_ref and u8_rec both given or both null)");
    const int rows = ceil_div(H, nbands);  // bands past the last row (nbands > ceil(H / rows)) write 0
    const dim3 grid(nbands, B);
    if (rec_dtype == VTP_F32)
        recon_pixels_kernel<float><<<grid, 256, 0, (cudaStream_t)st>>>(x, (const float*)rec, H, W, sub3, div3, rows, u8_ref,
                                                                      u8_rec, lp, sse_part);
    else
        recon_pixels_kernel<__nv_bfloat16><<<grid, 256, 0, (cudaStream_t)st>>>(x, (const __nv_bfloat16*)rec, H, W, sub3, div3,
                                                                              rows, u8_ref, u8_rec, lp, sse_part);
    VTP_LAUNCH_CHECK();
    return VTP_OK;
}

extern "C" int vtp_recon_ssim(const float* x, const void* rec, int rec_dtype, int B, int H, int W, const float* sub3,
                              const float* div3, double* part, vtp_stream_t st) {
    VTP_CHECK_ARG(x && rec && sub3 && div3 && part && B > 0 && B <= 65535 && H >= 11 && W >= 11 &&
                      (rec_dtype == VTP_F32 || rec_dtype == VTP_BF16),
                  "recon_ssim: bad args (H, W >= 11 for an 11x11 window)");
    const dim3 grid(ceil_div(W - 10, SSIM_TILE), ceil_div(H - 10, SSIM_TILE), B);
    if (rec_dtype == VTP_F32)
        recon_ssim_kernel<float><<<grid, 256, 0, (cudaStream_t)st>>>(x, (const float*)rec, H, W, sub3, div3, part);
    else
        recon_ssim_kernel<__nv_bfloat16><<<grid, 256, 0, (cudaStream_t)st>>>(x, (const __nv_bfloat16*)rec, H, W, sub3, div3,
                                                                            part);
    VTP_LAUNCH_CHECK();
    return VTP_OK;
}

extern "C" int vtp_recon_ssim_tiles(int H, int W) {
    if (H < 11 || W < 11) return 0;
    return ceil_div(W - 10, SSIM_TILE) * ceil_div(H - 10, SSIM_TILE);
}

extern "C" int vtp_recon_finalise(const double* sse_part, int nbands, const double* ssim_part, int ntiles,
                                  const double* lp_part, int nlp, int B, int H, int W, double* psnr, float* ssim,
                                  float* lpips, double* acc, vtp_stream_t st) {
    VTP_CHECK_ARG(sse_part && ssim_part && psnr && ssim && acc && B > 0 && H >= 11 && W >= 11 && nbands > 0 &&
                      ntiles == vtp_recon_ssim_tiles(H, W) && (!lp_part || (lpips && nlp > 0)),
                  "recon_finalise: bad args (ntiles must be vtp_recon_ssim_tiles(H, W))");
    const double npix = 3.0 * H * W, nwin = 3.0 * (H - 10) * (W - 10);
    recon_finalise_kernel<<<1, 256, 0, (cudaStream_t)st>>>(sse_part, nbands, ssim_part, ntiles, lp_part, nlp, B, npix, nwin,
                                                           psnr, ssim, lpips, acc);
    VTP_LAUNCH_CHECK();
    return VTP_OK;
}
