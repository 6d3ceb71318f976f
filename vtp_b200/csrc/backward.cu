// vtp_b200 — HBM-bound kernels of the training step: norm / SwiGLU / GELU / L2-normalise backward, bias-gradient
// column sums, gradient casts, embedding scatter, fused AdamW (+ bf16 weight refresh + EMA teacher).
// The reference publishes no training loop (SURVEY.md M3); these are the autograd duals of the forward stages in
// layers/normalization.py:17-22, layers/ffn.py:77-81, heads/dino_head.py:83-84, vtp.py:388-401 (EMA).
#include "host.h"
#include "ptx.cuh"

namespace vtp {

static inline int grid_cap(long n, int block) {
    long g = (n + block - 1) / block;
    long cap = (long)num_sms() * 16;
    return (int)(g < 1 ? 1 : (g < cap ? g : cap));
}

template <typename T>
__device__ __forceinline__ void ld4(const T* p, float (&v)[4]);
template <>
__device__ __forceinline__ void ld4<float>(const float* p, float (&v)[4]) {
    float4 t = *reinterpret_cast<const float4*>(p);
    v[0] = t.x, v[1] = t.y, v[2] = t.z, v[3] = t.w;
}
template <>
__device__ __forceinline__ void ld4<__nv_bfloat16>(const __nv_bfloat16* p, float (&v)[4]) {
    uint2 t = *reinterpret_cast<const uint2*>(p);
    v[0] = bf16_lo(t.x), v[1] = bf16_hi(t.x), v[2] = bf16_lo(t.y), v[3] = bf16_hi(t.y);
}

// ------------------------------------------------------------------------------------------------ norm backward
// g[m,:] += dx[m,:] where dx is the input-gradient of RMSNorm / LayerNorm given dy (bf16) ; dw += Σ dy∘xhat ; db += Σ dy
// One warp per row, 8 rows per warp-iteration strip; per-block column partials -> fp32 atomics.
// Occupancy: a 512-thread / 124-register version fits ONE block per SM (16 warps); 256-thread blocks capped at 80
// registers run three per SM; D <= 384 gets its own
// MAXV = 3 instantiation (36 column accumulators instead of 48) and the row values are re-derived from x, dy after the
// row reduction instead of being kept in a second register array.
template <typename TX, int MAXV>
__global__ void __launch_bounds__(256, (MAXV <= 4 ? 3 : (MAXV <= 8 ? 2 : 1))) norm_bwd_kernel(const TX* __restrict__ x, const float* __restrict__ rstd_, const float* __restrict__ mean_,
                                const float* __restrict__ w, const __nv_bfloat16* __restrict__ dy, float* __restrict__ g,
                                float* __restrict__ dw, float* __restrict__ db, int M, int D, int rows_per_block,
                                int is_ln, int x_rounded_bf16, __nv_bfloat16* __restrict__ gb_out,
                                float* __restrict__ gsum) {
    extern __shared__ float sred[];  // [3][D]: dw | db | column sums of the updated g
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
    for (int i = threadIdx.x; i < 3 * D; i += blockDim.x) sred[i] = 0.f;
    __syncthreads();
    float aw[MAXV][4], ab[MAXV][4], ag[MAXV][4];
#pragma unroll
    for (int gidx = 0; gidx < MAXV; ++gidx)
#pragma unroll
        for (int i = 0; i < 4; ++i) aw[gidx][i] = 0.f, ab[gidx][i] = 0.f, ag[gidx][i] = 0.f;
    // persistent blocks (round 2): a block walks strips blockIdx.x, blockIdx.x + gridDim.x, ... and flushes its column
    // partials ONCE — 444 blocks x 288 float4 atomics instead of one flush per 128-row strip (1 028 of them at M = 131 584,
    // 1 028-deep same-address chains in L2)
    const int nstrips = (M + rows_per_block - 1) / rows_per_block;
    for (int strip = blockIdx.x; strip < nstrips; strip += gridDim.x) {
    const int r0 = strip * rows_per_block;
    const int r1 = min(M, r0 + rows_per_block);
    for (int row = r0 + warp; row < r1; row += nw) {
        const float rstd = rstd_[row];
        const float mean = is_ln ? mean_[row] : 0.f;
        float xh[MAXV][4];   // normalised input; dy stays packed (bf16) and dy*w is re-derived after the row reduction
        uint2 dyp[MAXV];
        float4 gv4[MAXV];  // stream gradient: loaded up front so its latency overlaps the row reductions
        float s1 = 0.f, s2 = 0.f;
#pragma unroll
        for (int gidx = 0; gidx < MAXV; ++gidx) {
            const int c = (gidx * 32 + lane) * 4;
            if (c < D) {
                gv4[gidx] = *reinterpret_cast<const float4*>(g + (long)row * D + c);
                dyp[gidx] = *reinterpret_cast<const uint2*>(dy + (long)row * D + c);
            }
        }
#pragma unroll
        for (int gidx = 0; gidx < MAXV; ++gidx) {
            const int c = (gidx * 32 + lane) * 4;
            if (c < D) {
                float xv[4];
                ld4<TX>(x + (long)row * D + c, xv);
                const float dv[4] = {bf16_lo(dyp[gidx].x), bf16_hi(dyp[gidx].x), bf16_lo(dyp[gidx].y), bf16_hi(dyp[gidx].y)};
                const float4 w4 = __ldg(reinterpret_cast<const float4*>(w + c));
                const float wv[4] = {w4.x, w4.y, w4.z, w4.w};
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    float h = (xv[i] - mean) * rstd;
                    if (x_rounded_bf16) h = bf16_round(h);
                    xh[gidx][i] = h;
                    const float dx = dv[i] * wv[i];
                    s1 += dx;
                    s2 += dx * h;
                    aw[gidx][i] += dv[i] * h;
                    ab[gidx][i] += dv[i];
                }
            }
        }
        s1 = warp_sum(s1), s2 = warp_sum(s2);
        const float m1 = is_ln ? s1 / D : 0.f, m2 = s2 / D;
#pragma unroll
        for (int gidx = 0; gidx < MAXV; ++gidx) {
            const int c = (gidx * 32 + lane) * 4;
            if (c < D) {
                float4* gp = reinterpret_cast<float4*>(g + (long)row * D + c);
                float4 gv = gv4[gidx];
                const float4 w4 = __ldg(reinterpret_cast<const float4*>(w + c));
                gv.x += rstd * (bf16_lo(dyp[gidx].x) * w4.x - m1 - xh[gidx][0] * m2);
                gv.y += rstd * (bf16_hi(dyp[gidx].x) * w4.y - m1 - xh[gidx][1] * m2);
                gv.z += rstd * (bf16_lo(dyp[gidx].y) * w4.z - m1 - xh[gidx][2] * m2);
                gv.w += rstd * (bf16_hi(dyp[gidx].y) * w4.w - m1 - xh[gidx][3] * m2);
                *gp = gv;
                if (gb_out) {  // bf16 copy of the updated stream gradient = dY operand of the next (earlier) sub-layer
                    uint2 t2;
                    t2.x = pack_bf16x2(gv.x, gv.y), t2.y = pack_bf16x2(gv.z, gv.w);
                    *reinterpret_cast<uint2*>(gb_out + (long)row * D + c) = t2;
                }
                if (gsum) ag[gidx][0] += gv.x, ag[gidx][1] += gv.y, ag[gidx][2] += gv.z, ag[gidx][3] += gv.w;
            }
        }
    }
    }
#pragma unroll
    for (int gidx = 0; gidx < MAXV; ++gidx) {
        const int c = (gidx * 32 + lane) * 4;
        if (c < D) {
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                atomicAdd(&sred[c + i], aw[gidx][i]);
                if (is_ln) atomicAdd(&sred[D + c + i], ab[gidx][i]);
                if (gsum) atomicAdd(&sred[2 * D + c + i], ag[gidx][i]);
            }
        }
    }
    __syncthreads();
    for (int i = threadIdx.x * 4; i < D; i += blockDim.x * 4) {
        atomicAdd(reinterpret_cast<float4*>(dw + i), make_float4(sred[i], sred[i + 1], sred[i + 2], sred[i + 3]));
        if (is_ln && db)
            atomicAdd(reinterpret_cast<float4*>(db + i),
                      make_float4(sred[D + i], sred[D + i + 1], sred[D + i + 2], sred[D + i + 3]));
        if (gsum)
            atomicAdd(reinterpret_cast<float4*>(gsum + i),
                      make_float4(sred[2 * D + i], sred[2 * D + i + 1], sred[2 * D + i + 2], sred[2 * D + i + 3]));
    }
}

// ------------------------------------------------------------------------------------------------ SwiGLU / GELU backward
// Column-sum (bias-gradient) kernels: 2-D blocks (x = groups of columns, y = row lanes), each thread walks its rows of a
// ROWS_PER_BLOCK strip with several independent loads in flight, partial sums are reduced across y in shared memory
// and leave the block as ONE float4 atomic per 4 columns (same-address fp32 atomics serialise in a single L2 slice:
// the first version issued one per 32 rows and spent 2-4x the HBM time waiting on them).
static constexpr int CS_X = 128, CS_Y = 4;
static constexpr int CC_ROWS = 64;   // strip height of the persistent cast_colsum grid

template <int NF>  // NF floats of partial sums per thread
__device__ __forceinline__ void block_colsum_flush(float (&acc)[NF], float* sh /*[CS_Y][CS_X][NF]*/, float* dst, bool active) {
    float* mine = sh + ((threadIdx.y * CS_X + threadIdx.x) * NF);
#pragma unroll
    for (int i = 0; i < NF; ++i) mine[i] = acc[i];
    __syncthreads();
    if (threadIdx.y == 0 && active) {
#pragma unroll
        for (int i = 0; i < NF; i += 4) {
            float4 t = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
            for (int y = 0; y < CS_Y; ++y) {
                const float* o = sh + ((y * CS_X + threadIdx.x) * NF) + i;
                t.x += o[0], t.y += o[1], t.z += o[2], t.w += o[3];
            }
            atomicAdd(reinterpret_cast<float4*>(dst + i), t);
        }
    }
}

// pre packed [M][2Hs] (8-interleaved x1|x2, bf16), dhid [M][Hs] bf16 -> dpre [M][2Hs] bf16 ; dbias[2Hs] += colsum(dpre)
__global__ void __launch_bounds__(CS_X * CS_Y, 2)
swiglu_bwd_kernel(const __nv_bfloat16* __restrict__ pre, const __nv_bfloat16* __restrict__ dhid,
                  __nv_bfloat16* __restrict__ dpre, float* __restrict__ dbias, int M, int Hs) {
    __shared__ float sh[CS_Y * CS_X * 16];
    const int G = Hs / 8;
    const int gidx = blockIdx.x * CS_X + threadIdx.x;
    const bool active = gidx < G;
    float acc[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) acc[i] = 0.f;
    // persistent in y: the grid sweeps the rows CS_Y at a time (row-interleaved blocks, ONE loop: the strip form cost 14
    // registers and the second resident block), one flush of the bias-gradient partials per block
    if (active) {
        const int row_step = gridDim.y * CS_Y;
#pragma unroll 2
        for (int row = blockIdx.y * CS_Y + threadIdx.y; row < M; row += row_step) {
            const uint4 x1p = *reinterpret_cast<const uint4*>(pre + (long)row * 2 * Hs + 16 * gidx);
            const uint4 x2p = *reinterpret_cast<const uint4*>(pre + (long)row * 2 * Hs + 16 * gidx + 8);
            const uint4 dhp = *reinterpret_cast<const uint4*>(dhid + (long)row * Hs + 8 * gidx);
            const uint32_t x1w[4] = {x1p.x, x1p.y, x1p.z, x1p.w}, x2w[4] = {x2p.x, x2p.y, x2p.z, x2p.w};
            const uint32_t dhw[4] = {dhp.x, dhp.y, dhp.z, dhp.w};
            uint32_t o1[4], o2[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                float d1[2], d2[2];
#pragma unroll
                for (int hlf = 0; hlf < 2; ++hlf) {
                    const float x1 = hlf ? bf16_hi(x1w[k]) : bf16_lo(x1w[k]);
                    const float x2 = hlf ? bf16_hi(x2w[k]) : bf16_lo(x2w[k]);
                    const float dh = hlf ? bf16_hi(dhw[k]) : bf16_lo(dhw[k]);
                    const float sg = 1.f / (1.f + __expf(-x1));
                    d1[hlf] = dh * x2 * (sg * (1.f + x1 * (1.f - sg)));
                    d2[hlf] = dh * (x1 * sg);
                    acc[2 * k + hlf] += d1[hlf], acc[8 + 2 * k + hlf] += d2[hlf];
                }
                o1[k] = pack_bf16x2(d1[0], d1[1]), o2[k] = pack_bf16x2(d2[0], d2[1]);
            }
            *reinterpret_cast<uint4*>(dpre + (long)row * 2 * Hs + 16 * gidx) = make_uint4(o1[0], o1[1], o1[2], o1[3]);
            *reinterpret_cast<uint4*>(dpre + (long)row * 2 * Hs + 16 * gidx + 8) = make_uint4(o2[0], o2[1], o2[2], o2[3]);
        }
    }
    if (dbias) block_colsum_flush<16>(acc, sh, dbias + 16 * gidx, active);
}

// pre [M][N] bf16, dhid [M][N] bf16 -> dpre = dhid * gelu'(pre) ; dbias[N] += colsum(dpre)
__global__ void __launch_bounds__(CS_X * CS_Y, 2)
gelu_bwd_kernel(const __nv_bfloat16* __restrict__ pre, const __nv_bfloat16* __restrict__ dhid,
                __nv_bfloat16* __restrict__ dpre, float* __restrict__ dbias, int M, int N) {
    __shared__ float sh[CS_Y * CS_X * 8];
    const int G = N / 8;
    const int gidx = blockIdx.x * CS_X + threadIdx.x;
    const bool active = gidx < G;
    float acc[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] = 0.f;
    if (active) {
        const int row_step = gridDim.y * CS_Y;
#pragma unroll 2
        for (int row = blockIdx.y * CS_Y + threadIdx.y; row < M; row += row_step) {
            const uint4 xp = *reinterpret_cast<const uint4*>(pre + (long)row * N + 8 * gidx);
            const uint4 dp = *reinterpret_cast<const uint4*>(dhid + (long)row * N + 8 * gidx);
            const uint32_t xw[4] = {xp.x, xp.y, xp.z, xp.w}, dw[4] = {dp.x, dp.y, dp.z, dp.w};
            uint32_t o[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                float r[2];
#pragma unroll
                for (int hlf = 0; hlf < 2; ++hlf) {
                    const float xv = hlf ? bf16_hi(xw[k]) : bf16_lo(xw[k]);
                    const float dv = hlf ? bf16_hi(dw[k]) : bf16_lo(dw[k]);
                    const float cdf = 0.5f * (1.f + erff(xv * 0.70710678118654752f));
                    const float pdf = 0.3989422804014327f * __expf(-0.5f * xv * xv);
                    r[hlf] = dv * (cdf + xv * pdf);
                    acc[2 * k + hlf] += r[hlf];
                }
                o[k] = pack_bf16x2(r[0], r[1]);
            }
            *reinterpret_cast<uint4*>(dpre + (long)row * N + 8 * gidx) = make_uint4(o[0], o[1], o[2], o[3]);
        }
    }
    if (dbias) block_colsum_flush<8>(acc, sh, dbias + 8 * gidx, active);
}

// ------------------------------------------------------------------------------------------------ cast + column sum
// y bf16 [M][N] = (bf16) x[M][N] (TX fp32|bf16, row stride ldx) ; colsum[N] += Σ_m x  (bias gradient)
template <typename TX>
__global__ void __launch_bounds__(CS_X * CS_Y)
cast_colsum_kernel(const TX* __restrict__ x, long ldx, __nv_bfloat16* __restrict__ y, float* __restrict__ colsum, int M,
                   int N) {
    __shared__ float sh[CS_Y * CS_X * 4];
    const int G = N / 4;
    const int gidx = blockIdx.x * CS_X + threadIdx.x;
    const bool active = gidx < G;
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    // persistent in y (round 2): strips of CC_ROWS rows, one flush of the column partials per block
    const int nstrips = (M + CC_ROWS - 1) / CC_ROWS;
    if (active) {
        for (int strip = blockIdx.y; strip < nstrips; strip += gridDim.y) {
            const int r0 = strip * CC_ROWS, r1 = min(M, r0 + CC_ROWS);
#pragma unroll 4
            for (int row = r0 + threadIdx.y; row < r1; row += CS_Y) {
                float v[4];
                ld4<TX>(x + (long)row * ldx + 4 * gidx, v);
                acc[0] += v[0], acc[1] += v[1], acc[2] += v[2], acc[3] += v[3];
                if (y) {
                    uint2 t;
                    t.x = pack_bf16x2(v[0], v[1]), t.y = pack_bf16x2(v[2], v[3]);
                    *reinterpret_cast<uint2*>(y + (long)row * N + 4 * gidx) = t;
                }
            }
        }
    }
    if (colsum) block_colsum_flush<4>(acc, sh, colsum + 4 * gidx, active);
}

// ------------------------------------------------------------------------------------------------ L2-normalise backward
// y = x / max(||x||, eps):  dx = (dy − y (y·dy)) / max(||x||, eps).   One warp per row.
template <typename TY, typename TO>
__global__ void l2norm_bwd_kernel(const TY* __restrict__ y, const float* __restrict__ nrm, const float* __restrict__ dy,
                                  TO* __restrict__ dx, int M, int D, float eps) {
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (warp >= M) return;
    float dot = 0.f;
    for (int c = lane; c < D; c += 32) dot += (float)y[(long)warp * D + c] * dy[(long)warp * D + c];
    dot = warp_sum(dot);
    const float inv = 1.f / fmaxf(nrm[warp], eps);
    for (int c = lane; c < D; c += 32)
        dx[(long)warp * D + c] = (TO)((dy[(long)warp * D + c] - (float)y[(long)warp * D + c] * dot) * inv);
}

// ------------------------------------------------------------------------------------------------ scatter-add rows
// dst[idx[i]][:] += src[i][:] (fp32 atomics): token-embedding gradient, gather backward
template <typename TS>
__global__ void scatter_add_rows_kernel(const TS* __restrict__ src, long ld_src, float* __restrict__ dst, long ld_dst,
                                        const long long* __restrict__ idx, int n, int D) {
    const long total = (long)n * D;
    for (long t = blockIdx.x * (long)blockDim.x + threadIdx.x; t < total; t += (long)gridDim.x * blockDim.x) {
        const int d = (int)(t % D);
        const long i = t / D;
        atomicAdd(dst + idx[i] * ld_dst + d, (float)src[i * ld_src + d]);
    }
}

// ------------------------------------------------------------------------------------------------ fused AdamW (+EMA)
// p -= lr * (m̂ / (sqrt(v̂)+eps) + wd * p) on the fp32 master, refresh the bf16 compute copy in the same pass, and
// (optionally) the EMA teacher  t = mom*t + (1-mom)*p  (vtp.py:388-401) with its bf16 copy.  grad is scaled by
// gscale (1/world or loss scaling) and zeroed for the next step.
// `hyper` (optional, device): [0] step, [1] 1-b1^step, [2] 1-b2^step, [3] lr, [4] weight decay, [5] EMA momentum — written by
// hyper_tick_kernel so that a captured CUDA graph of the step needs no host-side scalars; it overrides the arguments.
__global__ void adamw_kernel(float* __restrict__ p, float* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
                             __nv_bfloat16* __restrict__ pb, float* __restrict__ tp, __nv_bfloat16* __restrict__ tpb,
                             long n4, float lr, float b1, float b2, float eps, float wd, float bc1, float bc2, float gscale,
                             float ema_mom, const float* __restrict__ hyper) {
    if (hyper) {
        bc1 = hyper[1], bc2 = hyper[2], lr = hyper[3], ema_mom = hyper[5];
        if (wd != 0.f) wd = hyper[4];     // regions without decay (norms, biases) keep 0
    }
    // 4 parameters per thread per iteration (all buffers are 128-byte aligned and n % 4 == 0 by construction).
    // The two divisions and the square root per parameter use the hardware approximations (MUFU.RCP / MUFU.SQRT, <= 2 ulp):
    // the IEEE sequences with their slow-path branches cost hundreds of instructions per float4, and the update is rounded
    // to a bf16 compute copy anyway.
    const float ibc1 = 1.f / bc1, ibc2 = 1.f / bc2;
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n4; i += (long)gridDim.x * blockDim.x) {
        float4 gi = reinterpret_cast<float4*>(g)[i];
        float4 mi = reinterpret_cast<float4*>(m)[i], vi = reinterpret_cast<float4*>(v)[i], pi = reinterpret_cast<float4*>(p)[i];
        reinterpret_cast<float4*>(g)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
        float ga[4] = {gi.x * gscale, gi.y * gscale, gi.z * gscale, gi.w * gscale};
        float ma[4] = {mi.x, mi.y, mi.z, mi.w}, va[4] = {vi.x, vi.y, vi.z, vi.w}, pa[4] = {pi.x, pi.y, pi.z, pi.w};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            ma[k] = b1 * ma[k] + (1.f - b1) * ga[k];
            va[k] = b2 * va[k] + (1.f - b2) * ga[k] * ga[k];
            float sq;
            asm("sqrt.approx.f32 %0, %1;" : "=f"(sq) : "f"(va[k] * ibc2));
            pa[k] -= lr * (__fdividef(ma[k] * ibc1, sq + eps) + wd * pa[k]);
        }
        reinterpret_cast<float4*>(m)[i] = make_float4(ma[0], ma[1], ma[2], ma[3]);
        reinterpret_cast<float4*>(v)[i] = make_float4(va[0], va[1], va[2], va[3]);
        reinterpret_cast<float4*>(p)[i] = make_float4(pa[0], pa[1], pa[2], pa[3]);
        if (pb) {
            uint2 w;
            w.x = pack_bf16x2(pa[0], pa[1]), w.y = pack_bf16x2(pa[2], pa[3]);
            reinterpret_cast<uint2*>(pb)[i] = w;
        }
        if (tp) {
            const float4 ti = reinterpret_cast<float4*>(tp)[i];
            float ta[4] = {ti.x, ti.y, ti.z, ti.w};
#pragma unroll
            for (int k = 0; k < 4; ++k) ta[k] = ema_mom * ta[k] + (1.f - ema_mom) * pa[k];
            reinterpret_cast<float4*>(tp)[i] = make_float4(ta[0], ta[1], ta[2], ta[3]);
            if (tpb) {
                uint2 w;
                w.x = pack_bf16x2(ta[0], ta[1]), w.y = pack_bf16x2(ta[2], ta[3]);
                reinterpret_cast<uint2*>(tpb)[i] = w;
            }
        }
    }
}

// one thread: step += 1, Adam bias corrections, and the scheduled lr / weight decay / teacher momentum of this step taken
// from device tables (the reference's CosineScheduler is a precomputed table too: models/utils/text_utils.py:160-207;
// past the end of a table its last entry = final_value holds)
__global__ void hyper_tick_kernel(float* __restrict__ hyper, float b1, float b2, const float* __restrict__ lr_tab,
                                  const float* __restrict__ wd_tab, const float* __restrict__ mom_tab, int n_tab) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    const float step = hyper[0] + 1.f;     // exact in fp32 up to 2^24 steps
    hyper[0] = step;
    hyper[1] = 1.f - powf(b1, step);
    hyper[2] = 1.f - powf(b2, step);
    if (n_tab > 0) {
        const int it = min((int)step - 1, n_tab - 1);   // schedule[it] for the it-th (0-based) optimiser step
        if (lr_tab) hyper[3] = lr_tab[it];
        if (wd_tab) hyper[4] = wd_tab[it];
        if (mom_tab) hyper[5] = mom_tab[it];
    }
}

__global__ void cast_f32_bf16_kernel(const float* __restrict__ x, __nv_bfloat16* __restrict__ y, long n) {
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x)
        y[i] = __float2bfloat16_rn(x[i]);
}

// g fp32 [B*T][D] -> out bf16 [B*HW][D] skipping the prefix rows (patch-embed wgrad operand); also returns
// dcls[D] += Σ_b g[b*T + 0][:]
__global__ void strip_prefix_kernel(const float* __restrict__ g, __nv_bfloat16* __restrict__ out, float* __restrict__ dcls,
                                    int B, int T, int prefix, int D) {
    const int HW = T - prefix;
    const long total = (long)B * T * (D / 4);
    for (long t = blockIdx.x * (long)blockDim.x + threadIdx.x; t < total; t += (long)gridDim.x * blockDim.x) {
        const int c = (int)(t % (D / 4)) * 4;
        const long row = t / (D / 4);
        const int tok = (int)(row % T);
        const long b = row / T;
        const float4 v = *reinterpret_cast<const float4*>(g + row * D + c);
        if (tok < prefix) {
            if (dcls) {
                atomicAdd(dcls + tok * D + c, v.x), atomicAdd(dcls + tok * D + c + 1, v.y);
                atomicAdd(dcls + tok * D + c + 2, v.z), atomicAdd(dcls + tok * D + c + 3, v.w);
            }
        } else {
            uint2 w;
            w.x = pack_bf16x2(v.x, v.y), w.y = pack_bf16x2(v.z, v.w);
            *reinterpret_cast<uint2*>(out + (b * HW + tok - prefix) * D + c) = w;
        }
    }
}

}  // namespace vtp

using namespace vtp;

extern "C" int vtp_norm_bwd(const void* x, int x_dtype, const float* rstd, const float* mean, const float* w, const void* dy,
                            float* g, float* dw, float* db, int M, int D, int is_ln, void* g_bf16_out, float* g_colsum,
                            vtp_stream_t st) {
    VTP_CHECK_ARG(x && rstd && w && dy && g && dw && M > 0, "norm_bwd: bad args");
    VTP_CHECK_ARG(D % 4 == 0 && D <= 2048, "norm_bwd: D %% 4 == 0 and D <= 2048");
    VTP_CHECK_ARG(!is_ln || mean, "norm_bwd: LayerNorm needs mean");
    VTP_CHECK_ARG((reinterpret_cast<uintptr_t>(dw) & 15) == 0 && (!db || (reinterpret_cast<uintptr_t>(db) & 15) == 0),
                  "norm_bwd: dw/db must be 16B aligned");
    const int threads = 256, rows_per_block = 32;    // strips of 32 rows (4 per warp), walked by a persistent grid
    const int per_sm = D <= 512 ? 3 : (D <= 1024 ? 2 : 1);   // resident blocks per SM (launch bounds of the MAXV variant)
    const int nstrips = ceil_div(M, rows_per_block);
    const int grid = nstrips < per_sm * num_sms() ? nstrips : per_sm * num_sms();
    VTP_CHECK_ARG(!g_colsum || (reinterpret_cast<uintptr_t>(g_colsum) & 15) == 0, "norm_bwd: g_colsum must be 16B aligned");
    const size_t smem = 3 * (size_t)D * sizeof(float);
    cudaStream_t s = (cudaStream_t)st;
    const int xr = (x_dtype == VTP_BF16 && !is_ln) ? 1 : 0;  // RMSNorm .type_as(x) rounding of xhat
#define LB(T, MV) \
    norm_bwd_kernel<T, MV><<<grid, threads, smem, s>>>((const T*)x, rstd, mean, w, (const __nv_bfloat16*)dy, g, dw, db, M, D, rows_per_block, is_ln, xr, (__nv_bfloat16*)g_bf16_out, g_colsum)
    if (x_dtype == VTP_F32) {
        if (D <= 384) LB(float, 3);
        else if (D <= 512) LB(float, 4);
        else if (D <= 768) LB(float, 6);
        else if (D <= 1024) LB(float, 8);
        else LB(float, 16);
    } else {
        if (D <= 384) LB(__nv_bfloat16, 3);
        else if (D <= 512) LB(__nv_bfloat16, 4);
        else if (D <= 768) LB(__nv_bfloat16, 6);
        else if (D <= 1024) LB(__nv_bfloat16, 8);
        else LB(__nv_bfloat16, 16);
    }
#undef LB
    VTP_LAUNCH_CHECK();
    return VTP_OK;
}

extern "C" int vtp_swiglu_bwd(const void* pre, const void* dhid, void* dpre, float* dbias, int M, int Hs, vtp_stream_t st) {
    VTP_CHECK_ARG(pre && dhid && dpre && M > 0 && Hs % 8 == 0, "swiglu_bwd: bad args");
    VTP_CHECK_ARG(!dbias || (reinterpret_cast<uintptr_t>(dbias) & 15) == 0, "swiglu_bwd: dbias must be 16B aligned");
    const int gx = ceil_div(Hs / 8, CS_X), groups = ceil_div(M, CS_Y);
    const int gy_cap = (2 * num_sms() + gx - 1) / gx;          // 2 resident 512-thread blocks per SM (64 registers): one wave
    dim3 grid(gx, groups < gy_cap ? groups : gy_cap), block(CS_X, CS_Y);
    swiglu_bwd_kernel<<<grid, block, 0, (cudaStream_t)st>>>((const __nv_bfloat16*)pre, (const __nv_bfloat16*)dhid,
                                                            (__nv_bfloat16*)dpre, dbias, M, Hs);
    VTP_LAUNCH_CHECK();
    return VTP_OK;
}

extern "C" int vtp_gelu_bwd(const void* pre, const void* dhid, void* dpre, float* dbias, int M, int N, vtp_stream_t st) {
    VTP_CHECK_ARG(pre && dhid && dpre && M > 0 && N % 8 == 0, "gelu_bwd: bad args");
    VTP_CHECK_ARG(!dbias || (reinterpret_cast<uintptr_t>(dbias) & 15) == 0, "gelu_bwd: dbias must be 16B aligned");
    const int gx = ceil_div(N / 8, CS_X), groups = ceil_div(M, CS_Y);
    const int gy_cap = (2 * num_sms() + gx - 1) / gx;
    dim3 grid(gx, groups < gy_cap ? groups : gy_cap), block(CS_X, CS_Y);
    gelu_bwd_kernel<<<grid, block, 0, (cudaStream_t)st>>>((const __nv_bfloat16*)pre, (const __nv_bfloat16*)dhid,
                                                          (__nv_bfloat16*)dpre, dbias, M, N);
    VTP_LAUNCH_CHECK();
    return VTP_OK;
}

extern "C" int vtp_cast_colsum(const void* x, int x_dtype, long ldx, void* y_bf16, float* colsum, int M, int N,
                               vtp_stream_t st) {
    VTP_CHECK_ARG(x && M > 0 && N % 4 == 0 && (y_bf16 || colsum), "cast_colsum: bad args");
    VTP_CHECK_ARG(!colsum || (reinterpret_cast<uintptr_t>(colsum) & 15) == 0, "cast_colsum: colsum must be 16B aligned");
    const int gx = ceil_div(N / 4, CS_X), strips = ceil_div(M, CC_ROWS);
    const int gy_cap = (4 * num_sms() + gx - 1) / gx;          // ~4 resident 512-thread blocks per SM in total
    dim3 grid(gx, strips < gy_cap ? strips : gy_cap), block(CS_X, CS_Y);
    if (x_dtype == VTP_F32)
        cast_colsum_kernel<float><<<grid, block, 0, (cudaStream_t)st>>>((const float*)x, ldx, (__nv_bfloat16*)y_bf16, colsum,
                                                                       M, N);
    else
        cast_colsum_kernel<__nv_bfloat16><<<grid, block, 0, (cudaStream_t)st>>>((const __nv_bfloat16*)x, ldx,
                                                                               (__nv_bfloat16*)y_bf16, colsum, M, N);
    VTP_LAUNCH_CHECK();
    return VTP_OK;
}

extern "C" int vtp_l2norm_bwd(const void* y, int y_dtype, const float* nrm, const float* dy, void* dx, int dx_dtype, int M,
                              int D, float eps, vtp_stream_t st) {
    VTP_CHECK_ARG(y && nrm && dy && dx && M > 0, "l2norm_bwd: bad args");
    const int grid = ceil_div(M, 8);
    cudaStream_t s = (cudaStream_t)st;
    if (y_dtype == VTP_F32 && dx_dtype == VTP_F32)
        l2norm_bwd_kernel<float, float><<<grid, 256, 0, s>>>((const float*)y, nrm, dy, (float*)dx, M, D, eps);
    else if (y_dtype == VTP_F32)
        l2norm_bwd_kernel<float, __nv_bfloat16><<<grid, 256, 0, s>>>((const float*)y, nrm, dy, (__nv_bfloat16*)dx, M, D, eps);
    else if (dx_dtype == VTP_F32)
        l2norm_bwd_kernel<__nv_bfloat16, float><<<grid, 256, 0, s>>>((const __nv_bfloat16*)y, nrm, dy, (float*)dx, M, D, eps);
    else
        l2norm_bwd_kernel<__nv_bfloat16, __nv_bfloat16>
            <<<grid, 256, 0, s>>>((const __nv_bfloat16*)y, nrm, dy, (__nv_bfloat16*)dx, M, D, eps);
    VTP_LAUNCH_CHECK();
    return VTP_OK;
}

extern "C" int vtp_scatter_add_rows(const void* src, int src_dtype, long ld_src, float* dst, long ld_dst, const int64_t* idx,
                                    int n, int D, vtp_stream_t st) {
    VTP_CHECK_ARG(src && dst && (idx || n == 0), "scatter_add_rows: bad args");
    if (n == 0) return VTP_OK;
    const long total = (long)n * D;
    if (src_dtype == VTP_F32)
        scatter_add_rows_kernel<float><<<grid_cap(total, 256), 256, 0, (cudaStream_t)st>>>((const float*)src, ld_src, dst,
                                                                                           ld_dst, (const long long*)idx, n, D);
    else
        scatter_add_rows_kernel<__nv_bfloat16><<<grid_cap(total, 256), 256, 0, (cudaStream_t)st>>>(
            (const __nv_bfloat16*)src, ld_src, dst, ld_dst, (const long long*)idx, n, D);
    VTP_LAUNCH_CHECK();
    return VTP_OK;
}

extern "C" int vtp_hyper_tick(float* hyper, float beta1, float beta2, const float* lr_tab, const float* wd_tab,
                              const float* mom_tab, int n_tab, vtp_stream_t st) {
    VTP_CHECK_ARG(hyper && n_tab >= 0 && (n_tab > 0 || (!lr_tab && !wd_tab && !mom_tab)), "hyper_tick: bad args");
    hyper_tick_kernel<<<1, 32, 0, (cudaStream_t)st>>>(hyper, beta1, beta2, lr_tab, wd_tab, mom_tab, n_tab);
    VTP_LAUNCH_CHECK();
    return VTP_OK;
}

extern "C" int vtp_adamw_step(float* p, float* g, float* m, float* v, void* p_bf16, float* teacher, void* teacher_bf16,
                              long n, float lr, float beta1, float beta2, float eps, float weight_decay, int step,
                              float grad_scale, float ema_momentum, const float* hyper, vtp_stream_t st) {
    VTP_CHECK_ARG(p && g && m && v && n > 0 && (step >= 1 || hyper), "adamw_step: bad args");
    VTP_CHECK_ARG(n % 4 == 0 && (reinterpret_cast<uintptr_t>(p) & 15) == 0 && (reinterpret_cast<uintptr_t>(g) & 15) == 0,
                  "adamw_step: n %% 4 == 0 and 16B-aligned buffers required");
    const float bc1 = 1.f - powf(beta1, (float)(step < 1 ? 1 : step)), bc2 = 1.f - powf(beta2, (float)(step < 1 ? 1 : step));
    adamw_kernel<<<grid_cap(n / 4, 256), 256, 0, (cudaStream_t)st>>>(p, g, m, v, (__nv_bfloat16*)p_bf16, teacher,
                                                                     (__nv_bfloat16*)teacher_bf16, n / 4, lr, beta1, beta2, eps,
                                                                     weight_decay, bc1, bc2, grad_scale, ema_momentum, hyper);
    VTP_LAUNCH_CHECK();
    return VTP_OK;
}

extern "C" int vtp_cast_f32_to_bf16(const float* x, void* y, long n, vtp_stream_t st) {
    VTP_CHECK_ARG(x && y && n > 0, "cast: bad args");
    cast_f32_bf16_kernel<<<grid_cap(n, 256), 256, 0, (cudaStream_t)st>>>(x, (__nv_bfloat16*)y, n);
    VTP_LAUNCH_CHECK();
    return VTP_OK;
}

extern "C" int vtp_strip_prefix(const float* g, void* out_bf16, float* dcls, int B, int T, int prefix, int D,
                                vtp_stream_t st) {
    VTP_CHECK_ARG(g && out_bf16 && B > 0 && D % 4 == 0 && prefix >= 0 && prefix < T, "strip_prefix: bad args");
    const long total = (long)B * T * (D / 4);
    strip_prefix_kernel<<<grid_cap(total, 256), 256, 0, (cudaStream_t)st>>>(g, (__nv_bfloat16*)out_bf16, dcls, B, T, prefix, D);
    VTP_LAUNCH_CHECK();
    return VTP_OK;
}

// ------------------------------------------------------------------------------------------------ weight norm
// heads/dino_head.py:48-49 (torch weight_norm, dim=0): W[k,:] = g[k] * v[k,:] / ||v[k,:]||
namespace vtp {
__global__ void weight_norm_fwd_kernel(const float* __restrict__ v, const float* __restrict__ g,
                                       __nv_bfloat16* __restrict__ w, float* __restrict__ vnorm, int K, int D) {
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (warp >= K) return;
    float s = 0.f;
    for (int c = lane; c < D; c += 32) {
        const float x = v[(long)warp * D + c];
        s += x * x;
    }
    s = warp_sum(s);
    const float nrm = sqrtf(s);
    if (lane == 0 && vnorm) vnorm[warp] = nrm;
    const float sc = g[warp] / nrm;
    for (int c = lane; c < D; c += 32) w[(long)warp * D + c] = __float2bfloat16_rn(v[(long)warp * D + c] * sc);
}
// dv += (g/||v||) (dW − (dW·v̂) v̂) ; dg += dW·v̂
__global__ void weight_norm_bwd_kernel(const float* __restrict__ v, const float* __restrict__ g,
                                       const float* __restrict__ vnorm, const float* __restrict__ dW,
                                       float* __restrict__ dv, float* __restrict__ dg, int K, int D) {
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (warp >= K) return;
    const float inv = 1.f / vnorm[warp];
    float dot = 0.f;
    for (int c = lane; c < D; c += 32) dot += dW[(long)warp * D + c] * v[(long)warp * D + c] * inv;
    dot = warp_sum(dot);
    const float sc = g[warp] * inv;
    for (int c = lane; c < D; c += 32)
        dv[(long)warp * D + c] += sc * (dW[(long)warp * D + c] - dot * v[(long)warp * D + c] * inv);
    if (lane == 0) dg[warp] += dot;
}
}  // namespace vtp

extern "C" int vtp_weight_norm_fwd(const float* v, const float* g, void* w_bf16, float* vnorm, int K, int D, vtp_stream_t st) {
    VTP_CHECK_ARG(v && g && w_bf16 && K > 0 && D > 0, "weight_norm_fwd: bad args");
    vtp::weight_norm_fwd_kernel<<<vtp::ceil_div(K, 8), 256, 0, (cudaStream_t)st>>>(v, g, (__nv_bfloat16*)w_bf16, vnorm, K, D);
    VTP_LAUNCH_CHECK();
    return VTP_OK;
}
extern "C" int vtp_weight_norm_bwd(const float* v, const float* g, const float* vnorm, const float* dW, float* dv, float* dg,
                                   int K, int D, vtp_stream_t st) {
    VTP_CHECK_ARG(v && g && vnorm && dW && dv && dg && K > 0, "weight_norm_bwd: bad args");
    vtp::weight_norm_bwd_kernel<<<vtp::ceil_div(K, 8), 256, 0, (cudaStream_t)st>>>(v, g, vnorm, dW, dv, dg, K, D);
    VTP_LAUNCH_CHECK();
    return VTP_OK;
}
