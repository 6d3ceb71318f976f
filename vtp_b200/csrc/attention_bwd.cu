// vtp_b200 — fused self-attention BACKWARD for short sequences (T = prefix + HW, prefix <= 1, HW <= 256) on wgmma.
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
    VTP_CHECK_ARG(B <= 65535, "attention_bwd: grid too large");
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
        configured = true;
    }
    const dim3 grid(H, p.pack ? ceil_div(B, p.pack) : B);
    if (p.nkt == 2) attn_bwd_kernel<2><<<grid, AB_THREADS, AB_SMEM, (cudaStream_t)st>>>(tq, td, p);
    else attn_bwd_kernel<1><<<grid, AB_THREADS, AB_SMEM, (cudaStream_t)st>>>(tq, td, p);
    VTP_LAUNCH_CHECK();
    return VTP_OK;
}
