// vtp_b200 — fused self-attention BACKWARD for short sequences (T = prefix + HW, prefix <= 1, HW <= 256) on wgmma.
// attn_bwd_kernel (below) holds a whole sequence in one CTA: packed tiles, HW <= 128, and causal HW <= 256.  Non-causal
// 128 < HW <= 256 (the 256² training step) runs attn_bwd_pair_kernel further down, a CTA pair per sequence.
//
// Gradient of layers/attention.py:110-126 (RoPE + SDPA) w.r.t. the packed pre-RoPE qkv projection output:
//   P = exp(s·QKᵀ − lse)      dV = Pᵀ dO      dP = dO Vᵀ      dS = s · P ∘ (dP − δ),  δ_i = Σ_d dO_id O_id
//   dQ = dS K                 dK = dSᵀ Q      then RoPEᵀ on dQ, dK (rotation is linear: layers/attention.py:12-23)
//
// All five GEMMs run on wgmma with the operands exactly as TMA lands them (128-row x 64-col bf16 tiles of Q, K, V out of
// the packed qkv buffer and of dO): the transposes are expressed through the wgmma transpose bits — Pᵀ / dSᵀ are MN-major
// A operands read from the same swizzled smem tile that serves dS as a K-major A operand for dQ; dO, Q, K are MN-major B
// operands.  The cls token (prefix) is handled on CUDA cores as in the forward kernel: as an extra key column by the row
// threads (rank-1 updates + a column reduction for dK_0/dV_0) and as an extra query row by a spare warp.
#include <stdlib.h>

#include "attention_bwd.cuh"
#include "host.h"
#include "ptx.cuh"

namespace vtp {

static constexpr int AB_THREADS = 384;  // 2 consumer warpgroups + warpgroup 2 (warp 8: TMA, cls query row)
static constexpr int BQ = 0, BK_ = 32768, BV = 65536, BDO = 98304, BP = 131072, BDS = 163840, BX = 196608;
// extras after BX: p0[264] | ds0[264] | dk0[64] | dv0[64] | pcol[2][128] | dscol[2][128] | barriers
static constexpr int X_P0 = 0, X_DS0 = 1056, X_DK0 = 2112, X_DV0 = 2368, X_PCOL = 2624, X_DSCOL = 3648, X_BAR = 4672;
static constexpr int AB_SMEM = BX + X_BAR + 128 + 1024;  // + alignment slack

struct AttnBwdDev {
    const __nv_bfloat16* qkv;   // [B*T][3D] post-RoPE q,k ; v
    const __nv_bfloat16* o;     // [B*T][D]
    const __nv_bfloat16* dout;  // [B*T][D]
    const float* lse;           // [B][H][T]
    __nv_bfloat16* dqkv;        // [B*T][3D] gradient w.r.t. the PRE-RoPE qkv
    const __nv_bfloat16* rope_sin;  // [HW][64] or null (no RoPE: text tower)
    const __nv_bfloat16* rope_cos;
    int B, T, H, D, prefix, HW, causal, nkt;
    float scale, scale_log2;
    // packed mode (T <= 64): `pack` whole sequences share the 128-row tile, their prefix tokens (`rprefix` per sequence)
    // are ordinary rows / key columns (prefix == 0 above) and P, dS are masked block-diagonally
    int pack, rprefix;
};

__device__ __forceinline__ void store_row64(__nv_bfloat16* g, const float (&f)[64]) {
    uint4* p = reinterpret_cast<uint4*>(g);
#pragma unroll
    for (int c = 0; c < 8; ++c) {
        uint4 w;
        w.x = pack_bf16x2(f[c * 8], f[c * 8 + 1]), w.y = pack_bf16x2(f[c * 8 + 2], f[c * 8 + 3]);
        w.z = pack_bf16x2(f[c * 8 + 4], f[c * 8 + 5]), w.w = pack_bf16x2(f[c * 8 + 6], f[c * 8 + 7]);
        p[c] = w;
    }
}
// dx = RoPEᵀ dy :  dx[i] = dy[i] cos[i] + dy[i+32] sin[i+32] ;  dx[i+32] = dy[i+32] cos[i+32] − dy[i] sin[i]
__device__ __forceinline__ void rope_bwd64(float (&g)[64], const __nv_bfloat16* sin_row, const __nv_bfloat16* cos_row) {
    float sn[64], cs[64];
    load_grow64(sin_row, sn);
    load_grow64(cos_row, cs);
#pragma unroll
    for (int i = 0; i < 32; ++i) {
        const float a = g[i], b = g[i + 32];
        g[i] = a * cs[i] + b * sn[i + 32];
        g[i + 32] = b * cs[i + 32] - a * sn[i];
    }
}

template <int NKT>
__global__ void __launch_bounds__(AB_THREADS, 1) attn_bwd_kernel(const __grid_constant__ CUtensorMap tm_qkv, const __grid_constant__ CUtensorMap tm_do,
                                                 const AttnBwdDev p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    float* p0 = reinterpret_cast<float*>(smem + BX + X_P0);
    float* ds0 = reinterpret_cast<float*>(smem + BX + X_DS0);
    float* dk0 = reinterpret_cast<float*>(smem + BX + X_DK0);
    float* dv0 = reinterpret_cast<float*>(smem + BX + X_DV0);
    float* pcol = reinterpret_cast<float*>(smem + BX + X_PCOL);
    float* dscol = reinterpret_cast<float*>(smem + BX + X_DSCOL);
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + BX + X_BAR);
    uint64_t* bar_ld = bars + 0;   // [2] tile loads
    uint64_t* bar_cls = bars + 2;  // p0/ds0 rows written by the cls warp

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int h = blockIdx.x, b = p.pack ? blockIdx.y * p.pack : blockIdx.y;
    const int D = p.D, T = p.T, prefix = p.prefix, HW = p.HW;
    const long row0 = (long)b * T;
    const int nkt = NKT;
    const float lse_l2 = 1.4426950408889634f;

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tm_qkv);
        tma_prefetch_desc(&tm_do);
        mbar_init(&bar_ld[0], 1), mbar_init(&bar_ld[1], 1), mbar_init(bar_cls, 1);
        fence_barrier_init();
    }
    if (threadIdx.x < 128) dk0[threadIdx.x & 63] = 0.f, dv0[threadIdx.x & 63] = 0.f;
    __syncthreads();

    if (warp < 8) {
        setmaxnreg_inc<200>();  // 384 x 168 registers: + 256 x 32 here = - 128 x 64 in warpgroup 2
        const int wg = warp >> 2, tw = threadIdx.x & 127, c4 = lane & 3;
        const uint32_t aQ = smem_u32(smem + BQ), aK = smem_u32(smem + BK_), aV = smem_u32(smem + BV);
        const uint32_t aDO = smem_u32(smem + BDO), aP = smem_u32(smem + BP), aDS = smem_u32(smem + BDS);
        int rr[2], pseq[2], ptok[2];
        bool pvalid[2];
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            rr[i] = 64 * wg + 16 * (tw >> 5) + (lane >> 2) + 8 * i;
            // packed mode: row r = token (r % T) of sequence b + r / T; it sees the key columns of its own sequence only
            pseq[i] = p.pack ? rr[i] / T : 0;
            pvalid[i] = p.pack && pseq[i] < p.pack && b + pseq[i] < p.B;
            ptok[i] = rr[i] - pseq[i] * T;
        }
        const __nv_bfloat16* kcls = p.qkv + row0 * 3 * D + D + h * 64;
        const __nv_bfloat16* vcls = p.qkv + row0 * 3 * D + 2 * D + h * 64;
        float lse_i[NKT][2], delta_i[NKT][2], ds_own[NKT][2];
        float dv[32], dk[32], dq[NKT][32];

#pragma unroll
        for (int n = 0; n < NKT * NKT; ++n) {
            const int kh = n / NKT, t = n % NKT;
            if (kh == 0) {
                // per-query-tile scalars (first visit of tile t): lse, delta = dO·O, and the cls-key column
                mbar_wait(&bar_ld[t], 0);
#pragma unroll
                for (int i = 0; i < 2; ++i) {
                    const int qi = 128 * t + rr[i];
                    const bool qvalid = p.pack ? pvalid[i] : qi < HW;
                    const long grow = row0 + prefix + qi;
                    lse_i[t][i] = 0.f, delta_i[t][i] = 0.f, ds_own[t][i] = 0.f;
                    float p0v = 0.f, ds0v = 0.f;
                    if (__any_sync(0xffffffffu, qvalid)) {  // quads are uniform: the shuffles stay inside valid quads
                        const float dl = quad_dot(smem + BDO + t * 16384, rr[i], p.o + (qvalid ? grow : row0) * D + h * 64, c4);
                        if (qvalid) {
                            lse_i[t][i] = p.pack ? p.lse[((long)(b + pseq[i]) * p.H + h) * T + ptok[i]]
                                                 : p.lse[((long)b * p.H + h) * T + prefix + qi];
                            delta_i[t][i] = dl;
                        }
                        if (prefix > 0) {
                            const float dp0 = quad_dot(smem + BDO + t * 16384, rr[i], vcls, c4);
                            const float s0 = quad_dot(smem + BQ + t * 16384, rr[i], kcls, c4);
                            if (qvalid) {
                                p0v = ex2f(s0 * p.scale_log2 - lse_i[t][i] * lse_l2);
                                ds0v = p.scale * p0v * (dp0 - dl);
                            }
                        }
                    }
                    ds_own[t][i] = ds0v;
                    if (prefix > 0 && c4 == 0) pcol[t * 128 + rr[i]] = p0v, dscol[t * 128 + rr[i]] = ds0v;
                }
                if (prefix > 0) {
                    // column reductions for the cls key: dV_0 += Σ_i p_i0 dO_i ; dK_0 += Σ_i ds_i0 q_i
                    asm volatile("bar.sync 1, 256;" ::: "memory");
                    if (threadIdx.x < 128) {
                        const int d = threadIdx.x & 63;
                        const bool isk = threadIdx.x >= 64;
                        const uint8_t* tile = smem + (isk ? BQ : BDO) + t * 16384;
                        const float* colv = (isk ? dscol : pcol) + t * 128;
                        float acc = 0.f;
                        for (int r = 0; r < 128; ++r)
                            acc = fmaf(colv[r], __uint_as_float((uint32_t)*reinterpret_cast<const uint16_t*>(tile + sw_off(r, d)) << 16), acc);
                        atomicAdd(isk ? &dk0[d] : &dv0[d], acc);
                    }
                }
            }
            if (n == 1 && NKT == 2) mbar_wait(&bar_ld[1], 0);
            // the P / dS tiles are free once both warpgroups have finished the previous step's MMAs
            asm volatile("bar.sync 1, 256;" ::: "memory");
#pragma unroll
            for (int c = 0; c < 2; ++c) {  // 64-key chunk c of key half kh
                float s[32], dpr[32];
                wgmma_fence();
#pragma unroll
                for (int j = 0; j < 4; ++j)
                    wgmma_m64n64_ss<0, 0>(s, wgmma_desc_sw128(aQ + t * 16384 + wg * 8192 + j * 32, 0, 1024),
                                          wgmma_desc_sw128(aK + kh * 16384 + c * 8192 + j * 32, 0, 1024), j > 0);
#pragma unroll
                for (int j = 0; j < 4; ++j)
                    wgmma_m64n64_ss<0, 0>(dpr, wgmma_desc_sw128(aDO + t * 16384 + wg * 8192 + j * 32, 0, 1024),
                                          wgmma_desc_sw128(aV + kh * 16384 + c * 8192 + j * 32, 0, 1024), j > 0);
                wgmma_commit();
                wgmma_wait<0>();
                fence_regs(s);
                fence_regs(dpr);
#pragma unroll
                for (int i = 0; i < 2; ++i) {
                    const int qi = 128 * t + rr[i];
                    const bool qvalid = p.pack ? pvalid[i] : qi < HW;
                    const int kmin = p.pack ? pseq[i] * T : 0;
                    const int kmax = p.pack ? kmin + T : (p.causal ? min(HW, qi + 1) : HW);
                    const float lsc = lse_i[t][i] * lse_l2, dl = delta_i[t][i];
#pragma unroll
                    for (int jn = 0; jn < 8; ++jn) {
                        const int key = 128 * kh + 64 * c + 8 * jn + 2 * c4;
                        float pe[2], de[2];
#pragma unroll
                        for (int cc = 0; cc < 2; ++cc) {
                            pe[cc] = 0.f, de[cc] = 0.f;
                            if (qvalid && key + cc >= kmin && key + cc < kmax) {
                                pe[cc] = ex2f(s[4 * jn + 2 * i + cc] * p.scale_log2 - lsc);
                                de[cc] = p.scale * pe[cc] * (dpr[4 * jn + 2 * i + cc] - dl);
                            }
                        }
                        const uint32_t off = c * 16384 + sw_off(rr[i], 8 * jn + 2 * c4);
                        *reinterpret_cast<uint32_t*>(smem + BP + off) = pack_bf16x2(pe[0], pe[1]);
                        *reinterpret_cast<uint32_t*>(smem + BDS + off) = pack_bf16x2(de[0], de[1]);
                    }
                }
            }
            fence_proxy_async_smem();
            asm volatile("bar.sync 1, 256;" ::: "memory");
            // P / dS tile: [128 q][128 keys] as 2 chunks of 64 keys.  As MN-major A (M = keys): chunk wg, K-step of 16
            // queries = 2048 B, SBO = 1024 (8 queries).  As K-major A (M = queries): k-step 32 B inside a chunk, next chunk
            // +16384, my 64 query rows +8192.
            wgmma_fence();
#pragma unroll
            for (int j = 0; j < 8; ++j) {  // reduction over 128 queries
                const uint64_t bdo = wgmma_desc_sw128(aDO + t * 16384 + j * 2048, 8192, 1024);
                const uint64_t bq = wgmma_desc_sw128(aQ + t * 16384 + j * 2048, 8192, 1024);
                wgmma_m64n64_ss<1, 1>(dv, wgmma_desc_sw128(aP + wg * 16384 + j * 2048, 8192, 1024), bdo, (t > 0 || j > 0));
                wgmma_m64n64_ss<1, 1>(dk, wgmma_desc_sw128(aDS + wg * 16384 + j * 2048, 8192, 1024), bq, (t > 0 || j > 0));
            }
#pragma unroll
            for (int j = 0; j < 8; ++j) {  // reduction over 128 keys
                const uint64_t ads = wgmma_desc_sw128(aDS + (j >> 2) * 16384 + wg * 8192 + (j & 3) * 32, 0, 1024);
                const uint64_t bk = wgmma_desc_sw128(aK + kh * 16384 + j * 2048, 8192, 1024);
                wgmma_m64n64_ss<0, 1>(dq[t], ads, bk, (kh > 0 || j > 0));
            }
            wgmma_commit();
            wgmma_wait<0>();
            fence_regs(dv);
            fence_regs(dk);
            fence_regs(dq[t]);

            if (t == NKT - 1) {
                // ------------ epilogue of key half kh: my key rows kj = 128 kh + rr[i]; acc[4 jn + 2 i + c] = dim 8 jn + 2 c4 + c
                if (prefix > 0) mbar_wait(bar_cls, 0);
#pragma unroll
                for (int i = 0; i < 2; ++i) {
                    const int kj = 128 * kh + rr[i];
                    if (!(p.pack ? pvalid[i] : kj < HW)) continue;
                    float gv[16], gk[16];
#pragma unroll
                    for (int e = 0; e < 16; ++e) {
                        const int jn = e >> 1, cc = e & 1;
                        gv[e] = dv[4 * jn + 2 * i + cc], gk[e] = dk[4 * jn + 2 * i + cc];
                    }
                    if (prefix > 0) {
                        const float pc = p0[kj], dc = ds0[kj];
                        const __nv_bfloat16* docls = p.dout + row0 * D + h * 64;  // dO of the cls query
                        const __nv_bfloat16* qc = p.qkv + row0 * 3 * D + h * 64;  // q of the cls query
#pragma unroll
                        for (int jn = 0; jn < 8; ++jn) {
                            const uint32_t wd = __ldg(reinterpret_cast<const uint32_t*>(docls + 8 * jn + 2 * c4));
                            const uint32_t wq = __ldg(reinterpret_cast<const uint32_t*>(qc + 8 * jn + 2 * c4));
                            gv[2 * jn] += pc * bf16_lo(wd), gv[2 * jn + 1] += pc * bf16_hi(wd);
                            gk[2 * jn] += dc * bf16_lo(wq), gk[2 * jn + 1] += dc * bf16_hi(wq);
                        }
                    }
                    const int pos = p.pack ? ptok[i] - p.rprefix : kj;  // patch position (prefix tokens are not rotated)
                    if (p.rope_sin && pos >= 0) rope_bwd_frag(gk, p.rope_sin + (long)pos * 64, p.rope_cos + (long)pos * 64, c4);
                    __nv_bfloat16* drow = p.dqkv + (row0 + prefix + kj) * 3 * D + h * 64;
#pragma unroll
                    for (int jn = 0; jn < 8; ++jn) {
                        *reinterpret_cast<uint32_t*>(drow + 2 * D + 8 * jn + 2 * c4) = pack_bf16x2(gv[2 * jn], gv[2 * jn + 1]);
                        *reinterpret_cast<uint32_t*>(drow + D + 8 * jn + 2 * c4) = pack_bf16x2(gk[2 * jn], gk[2 * jn + 1]);
                    }
                }
            }
        }
        // ------------ dQ epilogue of every query tile
#pragma unroll
        for (int t = 0; t < NKT; ++t) {
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                const int qi = 128 * t + rr[i];
                if (!(p.pack ? pvalid[i] : qi < HW)) continue;
                float gq[16];
#pragma unroll
                for (int e = 0; e < 16; ++e) gq[e] = dq[t][4 * (e >> 1) + 2 * i + (e & 1)];
                if (prefix > 0) {
#pragma unroll
                    for (int jn = 0; jn < 8; ++jn) {
                        const uint32_t w = __ldg(reinterpret_cast<const uint32_t*>(kcls + 8 * jn + 2 * c4));
                        gq[2 * jn] += ds_own[t][i] * bf16_lo(w), gq[2 * jn + 1] += ds_own[t][i] * bf16_hi(w);
                    }
                }
                const int pos = p.pack ? ptok[i] - p.rprefix : qi;
                if (p.rope_sin && pos >= 0) rope_bwd_frag(gq, p.rope_sin + (long)pos * 64, p.rope_cos + (long)pos * 64, c4);
                __nv_bfloat16* drow = p.dqkv + (row0 + prefix + qi) * 3 * D + h * 64;
#pragma unroll
                for (int jn = 0; jn < 8; ++jn)
                    *reinterpret_cast<uint32_t*>(drow + 8 * jn + 2 * c4) = pack_bf16x2(gq[2 * jn], gq[2 * jn + 1]);
            }
        }
    } else if (setmaxnreg_dec<104>(), warp == 8) {
        if (lane == 0) {
            // ------------------------------------------------ TMA: tile i = rows [128i, 128i+128) of Q,K,V,dO
            for (int i = 0; i < NKT; ++i) {
                const int r = (int)row0 + prefix + 128 * i;
                mbar_expect_tx(&bar_ld[i], 4 * 16384);
                tma_load_2d(smem + BQ + i * 16384, &tm_qkv, &bar_ld[i], h * 64, r);
                tma_load_2d(smem + BK_ + i * 16384, &tm_qkv, &bar_ld[i], D + h * 64, r);
                tma_load_2d(smem + BV + i * 16384, &tm_qkv, &bar_ld[i], 2 * D + h * 64, r);
                tma_load_2d(smem + BDO + i * 16384, &tm_do, &bar_ld[i], h * 64, r);
            }
        }
        __syncwarp();
        // ---------------------------------------------------- warp 8: the cls query row (prefix == 1)
        if (prefix > 0) {
            for (int i = 0; i < nkt; ++i) mbar_wait(&bar_ld[i], 0);
            float q0[64], do0[64];
            load_grow64(p.qkv + row0 * 3 * D + h * 64, q0);
            load_grow64(p.dout + row0 * D + h * 64, do0);
            float delta0 = 0.f;
            {
                float o0[64];
                load_grow64(p.o + row0 * D + h * 64, o0);
#pragma unroll
                for (int d = 0; d < 64; ++d) delta0 += do0[d] * o0[d];
            }
            const float lse0 = p.lse[((long)b * p.H + h) * T] * lse_l2;
            for (int i = 0; i < 8; ++i) {
                const int kj = lane + 32 * i;
                if (kj < 128 * nkt) {
                    float pv = 0.f, dsv = 0.f;
                    if (kj < HW) {
                        float f[64];
                        load_row64(smem + BK_, kj, f);  // K tiles are contiguous: row kj of [256][128B]
                        float s = 0.f;
#pragma unroll
                        for (int d = 0; d < 64; ++d) s += q0[d] * f[d];
                        load_row64(smem + BV, kj, f);
                        float dp = 0.f;
#pragma unroll
                        for (int d = 0; d < 64; ++d) dp += do0[d] * f[d];
                        pv = ex2f(s * p.scale_log2 - lse0);
                        dsv = p.scale * pv * (dp - delta0);
                    }
                    p0[kj] = pv, ds0[kj] = dsv;
                }
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(bar_cls);
            // cls-cls term
            float kc[64], vc[64];
            load_grow64(p.qkv + row0 * 3 * D + D + h * 64, kc);
            load_grow64(p.qkv + row0 * 3 * D + 2 * D + h * 64, vc);
            float s00 = 0.f, dp00 = 0.f;
#pragma unroll
            for (int d = 0; d < 64; ++d) s00 += q0[d] * kc[d], dp00 += do0[d] * vc[d];
            const float p00 = ex2f(s00 * p.scale_log2 - lse0);
            const float ds00 = p.scale * p00 * (dp00 - delta0);
            // dQ_0[d] = Σ_j ds_0j k_j[d] + ds_00 k_0[d]; lane owns dims 2*lane, 2*lane+1
            float a0 = 0.f, a1 = 0.f;
            for (int kj = 0; kj < HW; ++kj) {
                const float dsv = ds0[kj];
                const uint32_t w = *reinterpret_cast<const uint32_t*>(smem + BK_ + sw_off(kj, 2 * lane));
                a0 += dsv * bf16_lo(w), a1 += dsv * bf16_hi(w);
            }
            {
                const uint32_t w = __ldg(reinterpret_cast<const uint32_t*>(p.qkv + row0 * 3 * D + D + h * 64) + lane);
                a0 += ds00 * bf16_lo(w), a1 += ds00 * bf16_hi(w);
            }
            *reinterpret_cast<uint32_t*>(p.dqkv + row0 * 3 * D + h * 64 + 2 * lane) = pack_bf16x2(a0, a1);
            // stash p00/ds00 for the final dK_0/dV_0 write
            if (lane == 0) p0[260] = p00, ds0[260] = ds00;
        }
    }

    __syncthreads();
    if (warp == 8 && prefix > 0) {
        // dV_0 = Σ_i p_i0 dO_i (+ p_00 dO_0) ;  dK_0 = Σ_i ds_i0 q_i (+ ds_00 q_0)   — cls key row, no RoPE
        const float p00 = p0[260], ds00 = ds0[260];
        const uint32_t wdo = __ldg(reinterpret_cast<const uint32_t*>(p.dout + row0 * D + h * 64) + lane);
        const uint32_t wq = __ldg(reinterpret_cast<const uint32_t*>(p.qkv + row0 * 3 * D + h * 64) + lane);
        const float v0 = dv0[2 * lane] + p00 * bf16_lo(wdo), v1 = dv0[2 * lane + 1] + p00 * bf16_hi(wdo);
        const float k0 = dk0[2 * lane] + ds00 * bf16_lo(wq), k1 = dk0[2 * lane + 1] + ds00 * bf16_hi(wq);
        *reinterpret_cast<uint32_t*>(p.dqkv + row0 * 3 * D + 2 * D + h * 64 + 2 * lane) = pack_bf16x2(v0, v1);
        *reinterpret_cast<uint32_t*>(p.dqkv + row0 * 3 * D + D + h * 64 + 2 * lane) = pack_bf16x2(k0, k1);
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// attn_bwd_pair_kernel: non-causal, unpacked, 128 < HW <= 256.  A cluster of two CTAs per (head, image); CTA `rank` owns
// the 128 patch keys [128 rank, 128 rank + 128), 64 per consumer warpgroup, and walks the (up to) four 64-query tiles:
//   Sᵀ = K·Qᵀ, dPᵀ = V·dOᵀ (SS, K-major)   Pᵀ, dSᵀ in registers   dV += Pᵀ·dO, dK += dSᵀ·Q (RS, dO and Q MN-major)
//   dSᵀ (bf16) -> shared memory; warpgroup t % 2 then forms the CTA's partial dQ_t = dS_t·K over its 128 keys (SS, dS
//   read MN-major from both warpgroups' dSᵀ blocks) and parks it as fp32 in shared memory.
// After the last tile the pair sums its two partials through distributed shared memory (rank 0's + rank 1's, then the cls
// key column ds_i0 · k_0), rank t % 2 storing dQ_t.  Five patch GEMMs, no atomics, every element written by one thread.
// Warpgroup 2 (128 threads) streams the per-query scalars lse·log2e, δ = dO·O and ds_i0 into shared memory tile by tile
// and then, with a cls token, this rank's half of dQ_0, dK_0 and dV_0 (fp32, fixed order), which rank 0 completes and stores.
static constexpr int PR_K = 0, PR_V = 16384, PR_Q = 32768, PR_DO = 65536;  // K, V: 128 rows; Q, dO: 256 rows
static constexpr int PR_DS = 98304;   // [2 buffers][2 warpgroups] dSᵀ 64 keys x 64 queries, bf16 swizzled
static constexpr int PR_DQ = 131072;  // [4 tiles][8][128 threads] float4: partial dQ fragments
static constexpr int PR_SC = 196608;  // lse·log2e [256] | δ [256] | ds_i0 [256] | p_i0 [256] | lse_0·log2e, δ_0
static constexpr int PR_RED = PR_SC + 4352;  // [16 row groups][3][64] fp32 partial sums of dQ_0, dK_0, dV_0
static constexpr int PR_BAR = PR_RED + 16 * 3 * 64 * 4;
static constexpr int PR_SMEM = PR_BAR + 128 + 1024;  // + alignment slack

__device__ __forceinline__ float dot8(uint4 a, uint4 b) {  // 8-dim bf16 dot product
    return bf16_lo(a.x) * bf16_lo(b.x) + bf16_hi(a.x) * bf16_hi(b.x) + bf16_lo(a.y) * bf16_lo(b.y) +
           bf16_hi(a.y) * bf16_hi(b.y) + bf16_lo(a.z) * bf16_lo(b.z) + bf16_hi(a.z) * bf16_hi(b.z) +
           bf16_lo(a.w) * bf16_lo(b.w) + bf16_hi(a.w) * bf16_hi(b.w);
}
__device__ __forceinline__ float sum8(float x) {  // over the 8 lanes of an aligned lane group
    x += __shfl_xor_sync(0xffffffffu, x, 1);
    x += __shfl_xor_sync(0xffffffffu, x, 2);
    return x + __shfl_xor_sync(0xffffffffu, x, 4);
}
__device__ __forceinline__ void axpy8(float (&acc)[8], float w, uint4 x) {
    const uint32_t xs[4] = {x.x, x.y, x.z, x.w};
#pragma unroll
    for (int e = 0; e < 4; ++e) acc[2 * e] += w * bf16_lo(xs[e]), acc[2 * e + 1] += w * bf16_hi(xs[e]);
}

__global__ void __cluster_dims__(2, 1, 1) __launch_bounds__(AB_THREADS, 1)
    attn_bwd_pair_kernel(const __grid_constant__ CUtensorMap tm_qkv, const __grid_constant__ CUtensorMap tm_do,
                         const AttnBwdDev p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    float* lse_s = reinterpret_cast<float*>(smem + PR_SC);
    float* dl_s = lse_s + 256;
    float* dsc_s = lse_s + 512;
    float* psc_s = lse_s + 768;  // p_i0
    float* cls_s = lse_s + 1024;  // lse_0·log2e, δ_0
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + PR_BAR);
    uint64_t* bar_ld = bars;      // [2] K, V, Q / dO rows 0-127 ; Q / dO rows 128-255
    uint64_t* bar_sc = bars + 2;  // [4] scalars of query tile t written by the 4 warps of warpgroup 2

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int rank = (int)cluster_ctarank(), h = blockIdx.y, b = blockIdx.z;
    const int D = p.D, T = p.T, prefix = p.prefix, HW = p.HW;
    const long row0 = (long)b * T, lrow = ((long)b * p.H + h) * T;
    const int nqt = (HW + 63) / 64;
    const __nv_bfloat16* qcls = p.qkv + row0 * 3 * D + h * 64;  // cls token: q, k, v, dO
    const __nv_bfloat16* kcls = qcls + D;
    const __nv_bfloat16* vcls = qcls + 2 * D;
    const __nv_bfloat16* docls = p.dout + row0 * D + h * 64;

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tm_qkv);
        tma_prefetch_desc(&tm_do);
        mbar_init(&bar_ld[0], 1), mbar_init(&bar_ld[1], 1);
        for (int t = 0; t < 4; ++t) mbar_init(&bar_sc[t], 4);
        fence_barrier_init();
    }
    __syncthreads();

    if (warp < 8) {
        setmaxnreg_inc<200>();  // 384 x 168 registers: + 256 x 32 here = - 128 x 64 in warpgroup 2
        // broadcast so that ptxas sees the warpgroup index as warp-uniform: otherwise the dQ chain under `(t & 1) == wg`
        // is a divergent path and ptxas serialises every wgmma of the kernel (C7520)
        const int wg = __shfl_sync(0xffffffffu, warp >> 2, 0), tw = threadIdx.x & 127, c4 = lane & 3;
        int rr[2], kj[2];
        bool kvalid[2];
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            rr[i] = 64 * wg + 16 * (tw >> 5) + (lane >> 2) + 8 * i;  // key row in this CTA's K / V tiles
            kj[i] = 128 * rank + rr[i];
            kvalid[i] = kj[i] < HW;  // rows >= HW: the next image's rows or TMA zero fill
        }
        mbar_wait(&bar_ld[0], 0);
        mbar_wait(&bar_sc[0], 0);
        // the cls query row against my keys: p_0j, ds_0j (fp32, CUDA cores)
        float p0j[2] = {0.f, 0.f}, ds0j[2] = {0.f, 0.f};
        if (prefix > 0) {
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                const float s = quad_dot(smem + PR_K, rr[i], qcls, c4);
                const float dp = quad_dot(smem + PR_V, rr[i], docls, c4);
                if (kvalid[i]) {
                    p0j[i] = ex2f(s * p.scale_log2 - cls_s[0]);
                    ds0j[i] = p.scale * p0j[i] * (dp - cls_s[1]);
                }
            }
        }
        float dk[32], dv[32];
#pragma unroll
        for (int k = 0; k < 32; ++k) dk[k] = 0.f, dv[k] = 0.f;
        const uint32_t aK = smem_u32(smem + PR_K), aV = smem_u32(smem + PR_V);
#pragma unroll 1
        for (int t = 0; t < nqt; ++t) {
            if (t == 2) mbar_wait(&bar_ld[1], 0);
            mbar_wait(&bar_sc[t], 0);
            const uint32_t aQ = smem_u32(smem + PR_Q) + t * 8192, aDO = smem_u32(smem + PR_DO) + t * 8192;
            const uint32_t aDS = smem_u32(smem + PR_DS) + (t & 1) * 16384;
            float s[32], dp[32];  // Sᵀ, dPᵀ: rows = my keys, columns = the tile's 64 queries
            wgmma_fence();
#pragma unroll
            for (int j = 0; j < 4; ++j)
                wgmma_m64n64_ss<0, 0>(s, wgmma_desc_sw128(aK + wg * 8192 + j * 32, 0, 1024),
                                      wgmma_desc_sw128(aQ + j * 32, 0, 1024), j > 0);
#pragma unroll
            for (int j = 0; j < 4; ++j)
                wgmma_m64n64_ss<0, 0>(dp, wgmma_desc_sw128(aV + wg * 8192 + j * 32, 0, 1024),
                                      wgmma_desc_sw128(aDO + j * 32, 0, 1024), j > 0);
            wgmma_commit();
            wgmma_wait<0>();
            fence_regs(s);
            fence_regs(dp);
            const int qlim = HW - 64 * t;  // query columns >= qlim of this tile take no weight
#pragma unroll
            for (int jn = 0; jn < 8; ++jn)
#pragma unroll
                for (int c = 0; c < 2; ++c) {
                    const int qc = 8 * jn + 2 * c4 + c;
                    const float lq = lse_s[64 * t + qc], dq_ = dl_s[64 * t + qc];
#pragma unroll
                    for (int i = 0; i < 2; ++i) {
                        const int e = 4 * jn + 2 * i + c;
                        float pe = 0.f, de = 0.f;
                        if (kvalid[i] && qc < qlim) {
                            pe = ex2f(s[e] * p.scale_log2 - lq);
                            de = p.scale * pe * (dp[e] - dq_);
                        }
                        s[e] = pe, dp[e] = de;
                    }
                }
            uint32_t ap[4][4], as[4][4];
            pack_a(s, ap);
            pack_a(dp, as);
            // my dSᵀ block: 64 key rows x 64 query columns, row 16 (tw / 32) + lane / 4 + 8 i of block wg
            uint8_t* ds_blk = smem + PR_DS + (t & 1) * 16384 + wg * 8192;
#pragma unroll
            for (int kk = 0; kk < 4; ++kk)
#pragma unroll
                for (int q = 0; q < 4; ++q)
                    *reinterpret_cast<uint32_t*>(ds_blk + sw_off(rr[q & 1] - 64 * wg, 16 * kk + 8 * (q >> 1) + 2 * c4)) =
                        as[kk][q];
            fence_proxy_async_smem();
            wgmma_fence();
#pragma unroll
            for (int kk = 0; kk < 4; ++kk) {  // 16 queries per k-step, dO and Q as MN-major B operands
                wgmma_m64n64_rs<1>(dv, ap[kk], wgmma_desc_sw128(aDO + kk * 2048, 8192, 1024), 1);
                wgmma_m64n64_rs<1>(dk, as[kk], wgmma_desc_sw128(aQ + kk * 2048, 8192, 1024), 1);
            }
            wgmma_commit();
            // both dSᵀ blocks written; the buffer written next (tile t + 1) was last read by tile t - 1's dQ, complete
            asm volatile("bar.sync 1, 256;" ::: "memory");
            if ((t & 1) == wg) {
                float dq[32];
#pragma unroll
                for (int k = 0; k < 32; ++k) dq[k] = 0.f;
                // partial dQ_t = dS_t (64 q x 128 keys, MN-major: 16 keys = 2048 B) · K (128 keys x 64 dims, MN-major)
#pragma unroll
                for (int kk = 0; kk < 8; ++kk)
                    wgmma_m64n64_ss<1, 1>(dq, wgmma_desc_sw128(aDS + kk * 2048, 8192, 1024),
                                          wgmma_desc_sw128(aK + kk * 2048, 8192, 1024), kk > 0);
                wgmma_commit();
                wgmma_wait<0>();
                fence_regs(dq);
                float4* part = reinterpret_cast<float4*>(smem + PR_DQ + t * 16384);
#pragma unroll
                for (int k = 0; k < 8; ++k) part[k * 128 + tw] = make_float4(dq[4 * k], dq[4 * k + 1], dq[4 * k + 2], dq[4 * k + 3]);
            } else {
                wgmma_wait<0>();
            }
            fence_regs(dv);
            fence_regs(dk);
        }
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            if (!kvalid[i]) continue;
            const bool rope = p.rope_sin != nullptr;
            __nv_bfloat16* drow = p.dqkv + (row0 + prefix + kj[i]) * 3 * D + h * 64;
            store_grad_row(dv, i, p0j[i], prefix > 0 ? docls : nullptr, nullptr, nullptr, drow + 2 * D, c4);
            store_grad_row(dk, i, ds0j[i], prefix > 0 ? qcls : nullptr, rope ? p.rope_sin + (long)kj[i] * 64 : nullptr,
                           rope ? p.rope_cos + (long)kj[i] * 64 : nullptr, drow + D, c4);
        }
        // dQ of query tile t = rank + 2 wg: rank 0's partial + rank 1's partial, then the cls key column
        cluster_sync();
        const int t = rank + 2 * wg;
        if (t < nqt) {
            float dq[32];
            const uint32_t own = smem_u32(smem + PR_DQ + t * 16384) + tw * 16;
            const uint32_t peer = mapa_shared(own, (uint32_t)rank ^ 1u);
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                const float4 a = *reinterpret_cast<const float4*>(smem + PR_DQ + t * 16384 + (k * 128 + tw) * 16);
                const float4 r = ld_shared_cluster_f4(peer + k * 2048);
                dq[4 * k] = a.x + r.x, dq[4 * k + 1] = a.y + r.y, dq[4 * k + 2] = a.z + r.z, dq[4 * k + 3] = a.w + r.w;
            }
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                const int qi = 64 * t + 16 * (tw >> 5) + (lane >> 2) + 8 * i;
                if (qi >= HW) continue;
                const bool rope = p.rope_sin != nullptr;
                store_grad_row(dq, i, dsc_s[qi], prefix > 0 ? kcls : nullptr, rope ? p.rope_sin + (long)qi * 64 : nullptr,
                               rope ? p.rope_cos + (long)qi * 64 : nullptr,
                               p.dqkv + (row0 + prefix + qi) * 3 * D + h * 64, c4);
            }
        }
    } else {
        setmaxnreg_dec<104>();
        if (warp == 8 && lane == 0) {
            const int r = (int)row0 + prefix;
            mbar_expect_tx(&bar_ld[0], 4 * 16384);
            tma_load_2d(smem + PR_K, &tm_qkv, &bar_ld[0], D + h * 64, r + 128 * rank);
            tma_load_2d(smem + PR_V, &tm_qkv, &bar_ld[0], 2 * D + h * 64, r + 128 * rank);
            tma_load_2d(smem + PR_Q, &tm_qkv, &bar_ld[0], h * 64, r);
            tma_load_2d(smem + PR_DO, &tm_do, &bar_ld[0], h * 64, r);
            mbar_expect_tx(&bar_ld[1], 2 * 16384);
            tma_load_2d(smem + PR_Q + 16384, &tm_qkv, &bar_ld[1], h * 64, r + 128);
            tma_load_2d(smem + PR_DO + 16384, &tm_do, &bar_ld[1], h * 64, r + 128);
        }
        __syncwarp();
        // 8 threads per token row (16-byte chunk c = dims 8 c .. 8 c + 7), 16 rows per pass
        const int pt = threadIdx.x - 256, c = pt & 7, grp = pt >> 3;
        uint4 q0c = make_uint4(0, 0, 0, 0), do0c = q0c, k0c = q0c, v0c = q0c;
        float lse0 = 0.f, dl0 = 0.f;
        if (prefix > 0) {
            q0c = __ldg(reinterpret_cast<const uint4*>(qcls) + c), k0c = __ldg(reinterpret_cast<const uint4*>(kcls) + c);
            v0c = __ldg(reinterpret_cast<const uint4*>(vcls) + c), do0c = __ldg(reinterpret_cast<const uint4*>(docls) + c);
            dl0 = sum8(dot8(do0c, __ldg(reinterpret_cast<const uint4*>(p.o + row0 * D + h * 64) + c)));
            lse0 = p.lse[lrow] * LOG2E;
            if (pt == 0) cls_s[0] = lse0, cls_s[1] = dl0;
        }
        // pass 1, both ranks: the per-query scalars, tile by tile as the consumers need them
        for (int t = 0; t < nqt; ++t) {
#pragma unroll 4
            for (int ps = 0; ps < 4; ++ps) {
                const int q = 64 * t + 16 * ps + grp;
                const bool valid = q < HW;
                const long tok = row0 + prefix + (valid ? q : 0);
                const uint4 wd = __ldg(reinterpret_cast<const uint4*>(p.dout + tok * D + h * 64) + c);
                const uint4 wo = __ldg(reinterpret_cast<const uint4*>(p.o + tok * D + h * 64) + c);
                const float dl = sum8(dot8(wd, wo));
                const float lq = valid ? p.lse[lrow + prefix + q] * LOG2E : 0.f;
                float p_q0 = 0.f, ds_q0 = 0.f;  // query q against the cls key
                if (prefix > 0) {
                    const uint4 wq = __ldg(reinterpret_cast<const uint4*>(p.qkv + tok * 3 * D + h * 64) + c);
                    const float s_q0 = sum8(dot8(wq, k0c)), dp_q0 = sum8(dot8(wd, v0c));
                    p_q0 = valid ? ex2f(s_q0 * p.scale_log2 - lq) : 0.f;
                    ds_q0 = valid ? p.scale * p_q0 * (dp_q0 - dl) : 0.f;
                }
                if (c == 0) lse_s[q] = lq, dl_s[q] = valid ? dl : 0.f, dsc_s[q] = ds_q0, psc_s[q] = p_q0;
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&bar_sc[t]);
        }
        // pass 2, cls token: this rank's share (query / key tiles t = rank mod 2) of dQ_0 = Σ_j ds_0j k_j,
        // dK_0 = Σ_i ds_i0 q_i, dV_0 = Σ_i p_i0 dO_i, reduced over the 16 row groups in a fixed order
        float* red = reinterpret_cast<float*>(smem + PR_RED);  // [grp][dQ_0 | dK_0 | dV_0][64], then the sum [3][64]
        if (prefix > 0) {
            float aq[8], ak[8], av[8];
#pragma unroll
            for (int e = 0; e < 8; ++e) aq[e] = 0.f, ak[e] = 0.f, av[e] = 0.f;
            for (int t = rank; t < nqt; t += 2) {
#pragma unroll 2
                for (int ps = 0; ps < 4; ++ps) {
                    const int q = 64 * t + 16 * ps + grp;
                    const bool valid = q < HW;
                    const long tok = row0 + prefix + (valid ? q : 0);
                    const uint4* row = reinterpret_cast<const uint4*>(p.qkv + tok * 3 * D + h * 64);
                    const uint4 wq = __ldg(row + c), wk = __ldg(row + D / 8 + c), wv = __ldg(row + D / 4 + c);
                    const uint4 wd = __ldg(reinterpret_cast<const uint4*>(p.dout + tok * D + h * 64) + c);
                    const float s_0q = sum8(dot8(q0c, wk)), dp_0q = sum8(dot8(do0c, wv));
                    const float ds_0q = valid ? p.scale * ex2f(s_0q * p.scale_log2 - lse0) * (dp_0q - dl0) : 0.f;
                    axpy8(aq, ds_0q, wk);
                    axpy8(ak, dsc_s[q], wq);  // this row group's lane c = 0 wrote it in pass 1
                    axpy8(av, psc_s[q], wd);
                }
            }
#pragma unroll
            for (int e = 0; e < 8; ++e)
                red[grp * 192 + 8 * c + e] = aq[e], red[grp * 192 + 64 + 8 * c + e] = ak[e],
                                  red[grp * 192 + 128 + 8 * c + e] = av[e];
            asm volatile("bar.sync 2, 128;" ::: "memory");
            float x[3] = {0.f, 0.f, 0.f};
            if (pt < 64) {
                for (int g = 0; g < 16; ++g)
#pragma unroll
                    for (int v = 0; v < 3; ++v) x[v] += red[g * 192 + 64 * v + pt];
            }
            asm volatile("bar.sync 2, 128;" ::: "memory");
            if (pt < 64) red[pt] = x[0], red[64 + pt] = x[1], red[128 + pt] = x[2];
        }
        cluster_sync();
        if (prefix > 0 && rank == 0 && pt < 64) {
            // rank 0's share + rank 1's share, then the cls-cls term from the full 64-dim products
            const uint32_t peer = mapa_shared(smem_u32(red), 1u);
            float x[3];
#pragma unroll
            for (int v = 0; v < 3; ++v) {
                float r;
                asm volatile("ld.shared::cluster.f32 %0, [%1];" : "=f"(r) : "r"(peer + (64 * v + pt) * 4) : "memory");
                x[v] = red[64 * v + pt] + r;
            }
            float s00 = 0.f, dp00 = 0.f;
#pragma unroll
            for (int cc = 0; cc < 8; ++cc) {
                s00 += dot8(__ldg(reinterpret_cast<const uint4*>(qcls) + cc), __ldg(reinterpret_cast<const uint4*>(kcls) + cc));
                dp00 += dot8(__ldg(reinterpret_cast<const uint4*>(docls) + cc), __ldg(reinterpret_cast<const uint4*>(vcls) + cc));
            }
            const float p00 = ex2f(s00 * p.scale_log2 - lse0), ds00 = p.scale * p00 * (dp00 - dl0);
            const int d = pt;
            x[0] += ds00 * __bfloat162float(kcls[d]);
            x[1] += ds00 * __bfloat162float(qcls[d]);
            x[2] += p00 * __bfloat162float(docls[d]);
            __nv_bfloat16* drow = p.dqkv + row0 * 3 * D + h * 64 + d;
            drow[0] = __float2bfloat16_rn(x[0]), drow[D] = __float2bfloat16_rn(x[1]), drow[2 * D] = __float2bfloat16_rn(x[2]);
        }
    }
    cluster_sync();  // the peer's partial dQ stays readable until both CTAs are done with it
}

}  // namespace vtp

using namespace vtp;

extern "C" int vtp_attention_bwd(const void* qkv, const void* o, const void* dout, const float* lse, void* dqkv,
                                 const void* rope_sin, const void* rope_cos, int B, int T, int H, int prefix, int causal,
                                 vtp_stream_t st) {
    VTP_CHECK_ARG(qkv && o && dout && lse && dqkv && B > 0 && T > 0 && H > 0, "attention_bwd: bad args");
    VTP_CHECK_ARG(prefix == 0 || prefix == 1, "attention_bwd: prefix must be 0 or 1");
    VTP_CHECK_ARG(!(prefix && causal), "attention_bwd: causal + prefix is not supported");
    VTP_CHECK_ARG((rope_sin == nullptr) == (rope_cos == nullptr), "attention_bwd: rope tables");
    const int HW = T - prefix;
    VTP_CHECK_ARG(HW >= 1 && HW <= 256, "attention_bwd: %d non-prefix tokens not in [1,256]", HW);
    VTP_CHECK_ARG(B <= 65535 && H <= 65535, "attention_bwd: grid too large");
    const int D = H * 64;
    AttnBwdDev p;
    p.qkv = (const __nv_bfloat16*)qkv, p.o = (const __nv_bfloat16*)o, p.dout = (const __nv_bfloat16*)dout;
    p.lse = lse, p.dqkv = (__nv_bfloat16*)dqkv;
    p.rope_sin = (const __nv_bfloat16*)rope_sin, p.rope_cos = (const __nv_bfloat16*)rope_cos;
    p.B = B, p.T = T, p.H = H, p.D = D, p.prefix = prefix, p.HW = HW, p.causal = causal;
    p.nkt = HW > 128 ? 2 : 1;
    p.scale = 0.125f, p.scale_log2 = 0.125f * 1.4426950408889634f;
    p.pack = 0, p.rprefix = prefix;
    if (!causal && T <= 64 && B > 1 && getenv("VTP_ATTN_NO_PACK") == nullptr) {
        p.pack = 128 / T;
        p.prefix = 0, p.HW = T, p.nkt = 1;
    }
    CUtensorMap tq, td;
    {
        uint64_t dims[2] = {(uint64_t)3 * D, (uint64_t)B * T}, strides[1] = {(uint64_t)3 * D * 2};
        uint32_t box[2] = {64, 128};
        int rc = make_tmap_bf16(&tq, qkv, 2, dims, strides, box);
        if (rc) return rc;
    }
    {
        uint64_t dims[2] = {(uint64_t)D, (uint64_t)B * T}, strides[1] = {(uint64_t)D * 2};
        uint32_t box[2] = {64, 128};
        int rc = make_tmap_bf16(&td, dout, 2, dims, strides, box);
        if (rc) return rc;
    }
    static bool configured = false;
    if (!configured) {
        VTP_CUDA(cudaFuncSetAttribute(attn_bwd_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, AB_SMEM));
        VTP_CUDA(cudaFuncSetAttribute(attn_bwd_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, AB_SMEM));
        VTP_CUDA(cudaFuncSetAttribute(attn_bwd_pair_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, PR_SMEM));
        configured = true;
    }
    const dim3 grid(H, p.pack ? ceil_div(B, p.pack) : B);
    if (p.nkt == 2 && !causal) attn_bwd_pair_kernel<<<dim3(2, H, B), AB_THREADS, PR_SMEM, (cudaStream_t)st>>>(tq, td, p);
    else if (p.nkt == 2) attn_bwd_kernel<2><<<grid, AB_THREADS, AB_SMEM, (cudaStream_t)st>>>(tq, td, p);
    else attn_bwd_kernel<1><<<grid, AB_THREADS, AB_SMEM, (cudaStream_t)st>>>(tq, td, p);
    VTP_LAUNCH_CHECK();
    return VTP_OK;
}
