// vtp_b200 — non-causal self-attention forward for long sequences (T = prefix + HW, HW > 256): images above 256x256.
//
// Same op as attention.cu (layers/attention.py:110-126: SDPA with scale 1/sqrt(64), no mask) once the score row no
// longer fits the registers of one thread quad.
//
// bf16: one CTA per (query tile of 128 patch rows, head, image), like attn_fwd_kernel: two consumer warpgroups of 64
// query rows and one TMA producer warp.  The Q tile is loaded once; K and V 128-row tiles stream through an NSTAGE
// mbarrier ring (full: TMA landed, empty: all 8 consumer warps done with the stage).  Per key tile:
//   S = Q·Kᵀ      wgmma m64n128, K-major K straight out of the packed qkv buffer
//   online softmax in registers: running max / sum per row, O rescaled by exp2((m_old - m_new)·scale·log2e)
//   O += P·V      P re-packed in registers as the bf16 A operand, V consumed MN-major
// The prefix (cls) key columns are folded into each row's running softmax state on CUDA cores before the first tile,
// and the prefix query rows go to attn_prefix_rows_kernel (one CTA per row, all T keys from global memory).  This
// keeps the patch tiles 128-aligned: HW = 1024 is exactly 8 x 8 tiles.
//
// fp32 (accuracy mode): attn_fwd_f32_tiled_kernel, CUDA cores, one CTA per (64 query rows, head, image), K/V chunks of
// 128 keys in padded smem, online softmax with expf, no bf16 rounding anywhere.
#include "attention.h"
#include "host.h"
#include "ptx.cuh"

namespace vtp {

namespace {

constexpr int LONG_THREADS = 384;  // 2 consumer warpgroups + warpgroup 2 (warp 8 lane 0: TMA producer)
constexpr int NSTAGE = 3;
constexpr int TILE_BYTES = 128 * 128;  // 128 rows x 64 bf16
// smem: Q 16K | K stages | V stages | barriers (every tile 1024-aligned for the 128B swizzle)
constexpr int LQ = 0, LK = TILE_BYTES, LV = LK + NSTAGE * TILE_BYTES, LBAR = LV + NSTAGE * TILE_BYTES;
constexpr int LONG_SMEM = LBAR + 128 + 1024;  // + alignment slack

__device__ __forceinline__ float ex2f(float x) {  // ex2.approx.ftz (ex2f() carries a 4-instruction denormal slow path)
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
__device__ __forceinline__ uint32_t sw128_off(int row, int col /*bf16 element 0..63*/) {
    return row * 128 + ((((col >> 3) ^ (row & 7)) << 4) | ((col & 7) << 1));
}

__global__ void __launch_bounds__(LONG_THREADS, 1) attn_fwd_long_kernel(const __grid_constant__ CUtensorMap tm,
                                                                         const AttnDev p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + LBAR);
    uint64_t* bar_q = bars;                  // Q landed
    uint64_t* kfull = bars + 1;              // [NSTAGE] K tile landed
    uint64_t* vfull = kfull + NSTAGE;        // [NSTAGE] V tile landed
    uint64_t* empty = vfull + NSTAGE;        // [NSTAGE] stage released by the 8 consumer warps

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int qt = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
    const int D = p.D, prefix = p.prefix, HW = p.HW;
    const long seq_row0 = (long)b * p.T;
    const int nkt = (HW + 127) / 128;

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tm);
        mbar_init(bar_q, 1);
        for (int s = 0; s < NSTAGE; ++s) mbar_init(kfull + s, 1), mbar_init(vfull + s, 1), mbar_init(empty + s, 8);
        fence_barrier_init();
    }
    __syncthreads();

    if (warp < 8) {
        // ---------------- consumers: thread quad (lane / 4) of warp w owns query rows 16 w + lane / 4 (+ 8)
        setmaxnreg_inc<200>();
        const int wg = warp >> 2, tw = threadIdx.x & 127, c4 = lane & 3;
        int rr[2], qpos[2];
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            rr[i] = 64 * wg + 16 * (tw >> 5) + (lane >> 2) + 8 * i;  // row within the tile
            qpos[i] = 128 * qt + rr[i];                              // patch index of this query
        }
        mbar_wait(bar_q, 0);
        // running softmax state, seeded with the prefix key columns: m = max score, l = sum of exp2 numerators (this
        // thread's columns; quad-summed at the end), o = P·V with bf16-rounded numerators like the wgmma path
        float m[2], l[2], o[32];
#pragma unroll
        for (int k = 0; k < 32; ++k) o[k] = 0.f;
        {
            float s_pre[2][ATT_MAX_PREFIX];
#pragma unroll
            for (int j = 0; j < ATT_MAX_PREFIX; ++j) {
                float acc0 = 0.f, acc1 = 0.f;
                if (j < prefix) {
                    const uint4* kp = reinterpret_cast<const uint4*>(p.qkv + (seq_row0 + j) * 3 * D + D + h * 64 + 16 * c4);
#pragma unroll
                    for (int c = 0; c < 2; ++c) {
                        const uint4 w = __ldg(kp + c);
                        const uint4 q0 = *reinterpret_cast<const uint4*>(smem + LQ + sw128_off(rr[0], 16 * c4 + 8 * c));
                        const uint4 q1 = *reinterpret_cast<const uint4*>(smem + LQ + sw128_off(rr[1], 16 * c4 + 8 * c));
                        const uint32_t kw[4] = {w.x, w.y, w.z, w.w}, qw0[4] = {q0.x, q0.y, q0.z, q0.w},
                                       qw1[4] = {q1.x, q1.y, q1.z, q1.w};
#pragma unroll
                        for (int e = 0; e < 4; ++e) {
                            acc0 += bf16_lo(qw0[e]) * bf16_lo(kw[e]) + bf16_hi(qw0[e]) * bf16_hi(kw[e]);
                            acc1 += bf16_lo(qw1[e]) * bf16_lo(kw[e]) + bf16_hi(qw1[e]) * bf16_hi(kw[e]);
                        }
                    }
                }
                acc0 += __shfl_xor_sync(0xffffffffu, acc0, 1), acc1 += __shfl_xor_sync(0xffffffffu, acc1, 1);
                acc0 += __shfl_xor_sync(0xffffffffu, acc0, 2), acc1 += __shfl_xor_sync(0xffffffffu, acc1, 2);
                s_pre[0][j] = j < prefix ? acc0 : -INFINITY;
                s_pre[1][j] = j < prefix ? acc1 : -INFINITY;
            }
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                m[i] = -INFINITY;
                l[i] = 0.f;
#pragma unroll
                for (int j = 0; j < ATT_MAX_PREFIX; ++j) m[i] = fmaxf(m[i], s_pre[i][j]);
                const float msc = (m[i] == -INFINITY) ? 0.f : m[i] * p.scale_log2;
#pragma unroll
                for (int j = 0; j < ATT_MAX_PREFIX; ++j) {
                    if (j >= prefix) continue;
                    const float pe = ex2f(s_pre[i][j] * p.scale_log2 - msc);
                    if (c4 == 0) l[i] += pe;  // the prefix columns are counted once per row (quad sum below)
                    const float pb = bf16_round(pe);
                    const __nv_bfloat16* vp = p.qkv + (seq_row0 + j) * 3 * D + 2 * D + h * 64 + 2 * c4;
#pragma unroll
                    for (int jn = 0; jn < 8; ++jn) {
                        const uint32_t w = __ldg(reinterpret_cast<const uint32_t*>(vp + 8 * jn));
                        o[4 * jn + 2 * i] += pb * bf16_lo(w), o[4 * jn + 2 * i + 1] += pb * bf16_hi(w);
                    }
                }
            }
        }
        const uint32_t qa = smem_u32(smem + LQ) + wg * 8192;
        for (int t = 0; t < nkt; ++t) {
            const int st = t % NSTAGE;
            const uint32_t par = (t / NSTAGE) & 1;
            float s[64];
            mbar_wait(kfull + st, par);
            {
                const uint32_t ka = smem_u32(smem + LK + st * TILE_BYTES);
                wgmma_fence();
#pragma unroll
                for (int j = 0; j < 4; ++j)
                    wgmma_m64n128_ss<0, 0>(s, wgmma_desc_sw128(qa + j * 32, 0, 1024), wgmma_desc_sw128(ka + j * 32, 0, 1024),
                                           j > 0);
                wgmma_commit();
                wgmma_wait<0>();
                fence_regs(s);
            }
            // keys >= HW of the last tile (the next image's rows, or TMA zero fill past the buffer) take no weight;
            // score s[4 jn + 2 i + c] is key 8 jn + 2 c4 + c of row i
            const int klim = HW - 128 * t;
            if (klim < 128) {
#pragma unroll
                for (int jn = 0; jn < 16; ++jn)
#pragma unroll
                    for (int c = 0; c < 2; ++c)
                        if (8 * jn + 2 * c4 + c >= klim) s[4 * jn + c] = -INFINITY, s[4 * jn + 2 + c] = -INFINITY;
            }
            float mn[2] = {m[0], m[1]};
#pragma unroll
            for (int jn = 0; jn < 16; ++jn)
#pragma unroll
                for (int i = 0; i < 2; ++i) mn[i] = fmaxf(mn[i], fmaxf(s[4 * jn + 2 * i], s[4 * jn + 2 * i + 1]));
            float msc[2], alpha[2];
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                mn[i] = fmaxf(mn[i], __shfl_xor_sync(0xffffffffu, mn[i], 1));
                mn[i] = fmaxf(mn[i], __shfl_xor_sync(0xffffffffu, mn[i], 2));
                msc[i] = (mn[i] == -INFINITY) ? 0.f : mn[i] * p.scale_log2;
                alpha[i] = ex2f(m[i] * p.scale_log2 - msc[i]);  // m = -inf (no prefix, first tile) -> 0
                m[i] = mn[i];
                l[i] *= alpha[i];
            }
#pragma unroll
            for (int jn = 0; jn < 16; ++jn)
#pragma unroll
                for (int i = 0; i < 2; ++i)
#pragma unroll
                    for (int c = 0; c < 2; ++c) {
                        float& v = s[4 * jn + 2 * i + c];
                        v = ex2f(v * p.scale_log2 - msc[i]);  // masked -inf -> 0
                        l[i] += v;
                    }
#pragma unroll
            for (int jn = 0; jn < 8; ++jn)
#pragma unroll
                for (int i = 0; i < 2; ++i) o[4 * jn + 2 * i] *= alpha[i], o[4 * jn + 2 * i + 1] *= alpha[i];
            mbar_wait(vfull + st, par);
            {
                const uint32_t va = smem_u32(smem + LV + st * TILE_BYTES);
                wgmma_fence();
#pragma unroll
                for (int kk = 0; kk < 8; ++kk) {  // 16 keys per k-step
                    const uint32_t a[4] = {pack_bf16x2(s[8 * kk], s[8 * kk + 1]), pack_bf16x2(s[8 * kk + 2], s[8 * kk + 3]),
                                           pack_bf16x2(s[8 * kk + 4], s[8 * kk + 5]), pack_bf16x2(s[8 * kk + 6], s[8 * kk + 7])};
                    wgmma_m64n64_rs<1>(o, a, wgmma_desc_sw128(va + kk * 2048, 8192, 1024), 1);
                }
                wgmma_commit();
                wgmma_wait<0>();
                fence_regs(o);
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(empty + st);
        }
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            l[i] += __shfl_xor_sync(0xffffffffu, l[i], 1);
            l[i] += __shfl_xor_sync(0xffffffffu, l[i], 2);
        }
        // epilogue: o[4 jn + 2 i + c] is dim 8 jn + 2 c4 + c of row i; query rows >= HW are not stored
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            if (qpos[i] >= HW) continue;
            const float inv = 1.f / l[i];
            const long tok = seq_row0 + prefix + qpos[i];
            __nv_bfloat16* op = p.out + tok * D + h * 64 + 2 * c4;
#pragma unroll
            for (int jn = 0; jn < 8; ++jn)
                *reinterpret_cast<uint32_t*>(op + 8 * jn) = pack_bf16x2(o[4 * jn + 2 * i] * inv, o[4 * jn + 2 * i + 1] * inv);
            if (p.lse && c4 == 0) p.lse[((long)b * p.H + h) * p.T + prefix + qpos[i]] = m[i] * p.scale + logf(l[i]);
        }
    } else {
        setmaxnreg_dec<104>();
        if (warp != 8 || lane != 0) return;
        // ---------------- TMA producer
        const int row_k = (int)seq_row0 + prefix;
        mbar_expect_tx(bar_q, TILE_BYTES);
        tma_load_2d(smem + LQ, &tm, bar_q, h * 64, row_k + 128 * qt);
        for (int t = 0; t < nkt; ++t) {
            const int st = t % NSTAGE;
            if (t >= NSTAGE) mbar_wait(empty + st, ((t / NSTAGE) - 1) & 1);
            mbar_expect_tx(kfull + st, TILE_BYTES);
            tma_load_2d(smem + LK + st * TILE_BYTES, &tm, kfull + st, D + h * 64, row_k + 128 * t);
            mbar_expect_tx(vfull + st, TILE_BYTES);
            tma_load_2d(smem + LV + st * TILE_BYTES, &tm, vfull + st, 2 * D + h * 64, row_k + 128 * t);
        }
    }
}

// Prefix (cls) query rows of the long kernel: one CTA per (prefix row, head, image), its 8 warps take interleaved
// 32-key chunks of all T keys from global memory (online softmax per warp, fp32 accumulation, numerators rounded to
// bf16 before P·V as in attn_fwd_kernel's warp 8), then warp 0 merges the 8 partial states.
constexpr int PREFIX_WARPS = 8;

__global__ void __launch_bounds__(PREFIX_WARPS * 32) attn_prefix_rows_kernel(const AttnDev p) {
    __shared__ float sm_m[PREFIX_WARPS], sm_l[PREFIX_WARPS], sm_o[PREFIX_WARPS][64];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int j = blockIdx.x % p.prefix, h = (blockIdx.x / p.prefix) % p.H, b = blockIdx.x / (p.prefix * p.H);
    const int D = p.D, T = p.T;
    const long seq_row0 = (long)b * T;
    const long rs = 3L * D / 2;  // qkv row stride in bf16 pairs
    float qf[64];
    {
        const uint4* qp = reinterpret_cast<const uint4*>(p.qkv + (seq_row0 + j) * 3 * D + h * 64);
#pragma unroll
        for (int c = 0; c < 8; ++c) {
            const uint4 w = __ldg(qp + c);
            const uint32_t ww[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
            for (int e = 0; e < 4; ++e) qf[c * 8 + 2 * e] = bf16_lo(ww[e]), qf[c * 8 + 2 * e + 1] = bf16_hi(ww[e]);
        }
    }
    float m = -INFINITY, l = 0.f, a0 = 0.f, a1 = 0.f, c0 = 0.f, c1 = 0.f;
    for (int k0 = 32 * warp; k0 < T; k0 += 32 * PREFIX_WARPS) {
        const int k = k0 + lane;
        float s = -INFINITY;
        if (k < T) {
            const uint4* kp = reinterpret_cast<const uint4*>(p.qkv + (seq_row0 + k) * 3 * D + D + h * 64);
            float acc = 0.f;
#pragma unroll
            for (int c = 0; c < 8; ++c) {
                const uint4 w = __ldg(kp + c);
                const uint32_t ww[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
                for (int e = 0; e < 4; ++e) acc += qf[c * 8 + 2 * e] * bf16_lo(ww[e]) + qf[c * 8 + 2 * e + 1] * bf16_hi(ww[e]);
            }
            s = acc;
        }
        const float mn = fmaxf(m, warp_max(s));
        const float msc = mn * p.scale_log2;  // finite: key k0 is valid
        const float alpha = ex2f(m * p.scale_log2 - msc);
        m = mn;
        const float pe = (k < T) ? ex2f(s * p.scale_log2 - msc) : 0.f;
        l = l * alpha + pe;
        a0 *= alpha, a1 *= alpha, c0 *= alpha, c1 *= alpha;
        const float pb = bf16_round(pe);
        // O += P V: the lane owns output dims (2 lane, 2 lane + 1); two independent accumulator pairs, and a fully
        // unrolled full chunk so that its 32 V-row loads are in flight together
        const uint32_t* vp = reinterpret_cast<const uint32_t*>(p.qkv + (seq_row0 + k0) * 3 * D + 2 * D + h * 64) + lane;
        if (T - k0 >= 32) {
#pragma unroll
            for (int u = 0; u < 32; u += 2) {
                const float p0 = __shfl_sync(0xffffffffu, pb, u), p1 = __shfl_sync(0xffffffffu, pb, u + 1);
                const uint32_t w0 = __ldg(vp + u * rs), w1 = __ldg(vp + (u + 1) * rs);
                a0 += p0 * bf16_lo(w0), a1 += p0 * bf16_hi(w0);
                c0 += p1 * bf16_lo(w1), c1 += p1 * bf16_hi(w1);
            }
        } else {
            for (int u = 0; u < T - k0; ++u) {
                const float pu = __shfl_sync(0xffffffffu, pb, u);
                const uint32_t w = __ldg(vp + u * rs);
                a0 += pu * bf16_lo(w), a1 += pu * bf16_hi(w);
            }
        }
    }
    l = warp_sum(l);
    if (lane == 0) sm_m[warp] = m, sm_l[warp] = l;
    sm_o[warp][2 * lane] = a0 + c0, sm_o[warp][2 * lane + 1] = a1 + c1;
    __syncthreads();
    if (warp != 0) return;
    float M = -INFINITY;
#pragma unroll
    for (int w = 0; w < PREFIX_WARPS; ++w) M = fmaxf(M, sm_m[w]);
    float L = 0.f, o0 = 0.f, o1 = 0.f;
#pragma unroll
    for (int w = 0; w < PREFIX_WARPS; ++w) {
        const float f = (sm_m[w] == -INFINITY) ? 0.f : ex2f((sm_m[w] - M) * p.scale_log2);  // warp without keys: 0
        L += f * sm_l[w], o0 += f * sm_o[w][2 * lane], o1 += f * sm_o[w][2 * lane + 1];
    }
    const float inv = 1.f / L;
    *reinterpret_cast<uint32_t*>(p.out + (seq_row0 + j) * D + h * 64 + 2 * lane) = pack_bf16x2(o0 * inv, o1 * inv);
    if (p.lse && lane == 0) p.lse[((long)b * p.H + h) * T + j] = M * p.scale + logf(L);
}

// fp32 accuracy mode, T beyond the smem-resident kernel: CTA = (64 query rows, head, image), 8 warps x 8 rows; per
// 128-key chunk a lane scores keys lane + 32 i against the row's q (smem broadcast), then the warp accumulates P·V
// with the lane owning dims lane and lane + 32.
constexpr int F32_QROWS = 64, F32_KC = 128, F32_WARPS = 8, F32_RPW = F32_QROWS / F32_WARPS;
constexpr int F32_SMEM = (F32_KC * 65 + F32_KC * 64 + F32_QROWS * 64 + F32_WARPS * F32_KC) * (int)sizeof(float);

__global__ void __launch_bounds__(F32_WARPS * 32, 2) attn_fwd_f32_tiled_kernel(const float* __restrict__ qkv,
                                                                            float* __restrict__ out, int T, int H,
                                                                            float scale) {
    extern __shared__ float sm[];
    float* Ks = sm;                    // [KC][65]
    float* Vs = Ks + F32_KC * 65;      // [KC][64]
    float* Qs = Vs + F32_KC * 64;      // [QROWS][64]
    float* Ps = Qs + F32_QROWS * 64;   // [WARPS][KC]
    const int D = H * 64, q0 = blockIdx.x * F32_QROWS, h = blockIdx.y, b = blockIdx.z;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const float* base = qkv + (long)b * T * 3 * D;
    for (int i = threadIdx.x; i < F32_QROWS * 64; i += blockDim.x) {
        const int r = i >> 6, d = i & 63;
        Qs[i] = (q0 + r < T) ? base[(long)(q0 + r) * 3 * D + h * 64 + d] : 0.f;
    }
    float* pw = Ps + warp * F32_KC;
    float m[F32_RPW], l[F32_RPW], a0[F32_RPW], a1[F32_RPW];
#pragma unroll
    for (int r = 0; r < F32_RPW; ++r) m[r] = -INFINITY, l[r] = 0.f, a0[r] = 0.f, a1[r] = 0.f;
    for (int k0 = 0; k0 < T; k0 += F32_KC) {
        const int n = min(F32_KC, T - k0);
        __syncthreads();  // previous chunk fully consumed (and Qs written, first time round)
        for (int i = threadIdx.x; i < n * 64; i += blockDim.x) {
            const int t = i >> 6, d = i & 63;
            Ks[t * 65 + d] = base[(long)(k0 + t) * 3 * D + D + h * 64 + d];
            Vs[t * 64 + d] = base[(long)(k0 + t) * 3 * D + 2 * D + h * 64 + d];
        }
        __syncthreads();
#pragma unroll
        for (int r = 0; r < F32_RPW; ++r) {
            const float* qr = Qs + (warp * F32_RPW + r) * 64;
            float s[F32_KC / 32];
            float cm = -INFINITY;
#pragma unroll
            for (int i = 0; i < F32_KC / 32; ++i) {
                const int k = lane + 32 * i;
                s[i] = -INFINITY;
                if (k < n) {
                    float acc = 0.f;
#pragma unroll
                    for (int d = 0; d < 64; ++d) acc += qr[d] * Ks[k * 65 + d];
                    s[i] = acc * scale;
                }
                cm = fmaxf(cm, s[i]);
            }
            const float mn = fmaxf(m[r], warp_max(cm));
            const float alpha = expf(m[r] - mn);  // m = -inf on the first chunk -> 0
            m[r] = mn;
            float ls = 0.f;
#pragma unroll
            for (int i = 0; i < F32_KC / 32; ++i) {
                const float e = (lane + 32 * i < n) ? expf(s[i] - mn) : 0.f;
                pw[lane + 32 * i] = e;
                ls += e;
            }
            l[r] = l[r] * alpha + ls;
            __syncwarp();
            float x0 = a0[r] * alpha, x1 = a1[r] * alpha;
            for (int k = 0; k < n; ++k) {
                const float pk = pw[k];
                x0 += pk * Vs[k * 64 + lane], x1 += pk * Vs[k * 64 + 32 + lane];
            }
            a0[r] = x0, a1[r] = x1;
            __syncwarp();
        }
    }
#pragma unroll
    for (int r = 0; r < F32_RPW; ++r) {
        const int q = q0 + warp * F32_RPW + r;
        if (q >= T) continue;
        const float lt = warp_sum(l[r]);
        float* op = out + ((long)b * T + q) * D + h * 64;
        op[lane] = a0[r] / lt, op[32 + lane] = a1[r] / lt;
    }
}

}  // namespace

int attn_fwd_long(const CUtensorMap& tm, const AttnDev& p, cudaStream_t st) {
    static bool configured = false;
    if (!configured) {
        VTP_CUDA(cudaFuncSetAttribute(attn_fwd_long_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, LONG_SMEM));
        configured = true;
    }
    attn_fwd_long_kernel<<<dim3(ceil_div(p.HW, 128), p.H, p.B), LONG_THREADS, LONG_SMEM, st>>>(tm, p);
    VTP_LAUNCH_CHECK();
    if (p.prefix > 0) {
        attn_prefix_rows_kernel<<<p.B * p.H * p.prefix, PREFIX_WARPS * 32, 0, st>>>(p);
        VTP_LAUNCH_CHECK();
    }
    return VTP_OK;
}

int attn_fwd_f32_tiled(const float* qkv, float* out, int B, int T, int H, cudaStream_t st) {
    static bool configured = false;
    if (!configured) {
        VTP_CUDA(cudaFuncSetAttribute(attn_fwd_f32_tiled_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, F32_SMEM));
        configured = true;
    }
    attn_fwd_f32_tiled_kernel<<<dim3(ceil_div(T, F32_QROWS), H, B), F32_WARPS * 32, F32_SMEM, st>>>(qkv, out, T, H,
                                                                                                   0.125f);
    VTP_LAUNCH_CHECK();
    return VTP_OK;
}

}  // namespace vtp
