// vtp_b200 — fused self-attention forward for short sequences (T = prefix + HW, HW <= 256) on wgmma.
//
// Replaces layers/attention.py:110-126 (SelfAttention.compute_attention after RoPE: SDPA with scale 1/sqrt(64), no
// mask, no dropout) and nn.MultiheadAttention's causal SDPA in the text tower (layers/block.py:387-412).
//
// HW <= 128 and the packed short sequences: attn_fwd_kernel, one CTA per (query tile of 128 patch rows, head, image):
// two consumer warpgroups of 64 query rows each and one extra warp.
//   S = Q·Kᵀ     one wgmma chain per warpgroup  m64 x N=128 x K=64  (Q,K tiles by TMA straight out of the packed qkv
//                buffer); the whole score row lives in the registers of one thread quad -> exact single-pass softmax
//   O = P·V      P is re-packed in registers as the bf16 A operand (no shared-memory round trip), V is consumed as an
//                MN-major B operand (no transpose)
// 128 < HW <= 256 (the 256² training step): attn_fwd_256_kernel below, 64-row CTAs, two 128-key halves.
// The `prefix` (cls / storage) tokens — 1 in the encoder, 0 in the decoder/text — would cost a third 128-row tile for
// one row, so they are handled on CUDA cores: their key columns are folded into every row's softmax by the row
// threads, and their query rows are computed from the K/V tiles already in smem (by the extra warp in
// attn_fwd_kernel, by the four warps of a CTA together in attn_fwd_256_kernel).
#include <stdlib.h>

#include "attention.h"
#include "host.h"
#include "ptx.cuh"

namespace vtp {

static constexpr int ATT_THREADS = 384;  // 2 consumer warpgroups + warpgroup 2 (warp 8: TMA, prefix query rows)
static constexpr int MAX_PREFIX = ATT_MAX_PREFIX;
// smem: Q 16K | K 16K | V 16K | barriers
static constexpr int SQ = 0, SK = 16384, SV = SK + 16384, SBAR = SV + 16384;
static constexpr int SPCLS = SBAR + 128;      // bf16 [256]: softmax numerators of the cls query row (warp 8)
static constexpr int ATT_SMEM = SPCLS + 512 + 1024;  // + alignment slack

__device__ __forceinline__ float ex2f(float x) {  // ex2.approx.ftz (ex2f() carries a 4-instruction denormal slow path)
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
__device__ __forceinline__ uint32_t sw128_off(int row, int col /*bf16 element 0..63*/) {
    return row * 128 + ((((col >> 3) ^ (row & 7)) << 4) | ((col & 7) << 1));
}

__global__ void __launch_bounds__(ATT_THREADS, 1) attn_fwd_kernel(const __grid_constant__ CUtensorMap tm, const AttnDev p) {
    constexpr int NK = 128;  // key columns of S
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + SBAR);
    uint64_t* bar_qk = bars + 0;  // Q,K landed
    uint64_t* bar_v = bars + 1;   // V landed

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    // packed mode (short sequences, e.g. the 37-token local crops): the tile holds `pack` consecutive sequences, every
    // token (cls included) is an ordinary query row / key column and the softmax is masked block-diagonally
    const int qt = blockIdx.x, h = blockIdx.y, b = p.pack ? blockIdx.z * p.pack : blockIdx.z;
    const int D = p.D, T = p.T, prefix = p.prefix, HW = p.HW;
    const long seq_row0 = (long)b * T;
    const int kvrows = NK;

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tm);
        mbar_init(bar_qk, 1), mbar_init(bar_v, 1);
        fence_barrier_init();
    }
    __syncthreads();

    if (warp < 8) {
        // ---------------- consumers: thread quad (lane / 4) of warp w owns query rows 16 w + lane / 4 (+ 8)
        setmaxnreg_inc<200>();  // 384 x 168 registers: + 256 x 32 here = - 128 x 64 in warpgroup 2
        const int wg = warp >> 2, tw = threadIdx.x & 127, c4 = lane & 3;
        int rr[2], qpos[2], qtok[2], pseq[2], kmin[2], kmax[2];
        bool row_valid[2];
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            rr[i] = 64 * wg + 16 * (tw >> 5) + (lane >> 2) + 8 * i;  // row within the tile
            qpos[i] = 128 * qt + rr[i];                              // patch index of this query
            qtok[i] = prefix + qpos[i];                              // token index within the sequence
            pseq[i] = p.pack ? rr[i] / T : 0;                        // packed mode: my sequence within the tile
            row_valid[i] = p.pack ? (pseq[i] < p.pack && b + pseq[i] < p.B) : (qpos[i] < HW);
            // keys [kmin,kmax) are visible
            kmin[i] = p.pack ? (row_valid[i] ? pseq[i] * T : 0) : 0;
            kmax[i] = p.pack ? (row_valid[i] ? kmin[i] + T : 0) : (p.causal ? min(HW, qpos[i] + 1) : HW);
        }
        mbar_wait(bar_qk, 0);
        float s[NK / 2];
        {
            const uint32_t qa = smem_u32(smem + SQ) + wg * 8192, ka = smem_u32(smem + SK);
            wgmma_fence();
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const uint64_t ad = wgmma_desc_sw128(qa + j * 32, 0, 1024), bd = wgmma_desc_sw128(ka + j * 32, 0, 1024);
                wgmma_m64n128_ss<0, 0>(s, ad, bd, j > 0);
            }
            wgmma_commit();
        }
        // scores against the prefix keys (CUDA cores, while the MMAs run): q rows from smem (swizzled), k rows from
        // global; the four threads of the quad take 16 dims each
        float s_pre[2][MAX_PREFIX];
#pragma unroll
        for (int j = 0; j < MAX_PREFIX; ++j) {
            float acc0 = 0.f, acc1 = 0.f;
            if (j < prefix) {
                const uint4* kp = reinterpret_cast<const uint4*>(p.qkv + (seq_row0 + j) * 3 * D + D + h * 64 + 16 * c4);
#pragma unroll
                for (int c = 0; c < 2; ++c) {
                    const uint4 w = __ldg(kp + c);
                    const uint4 q0 = *reinterpret_cast<const uint4*>(smem + SQ + sw128_off(rr[0], 16 * c4 + 8 * c));
                    const uint4 q1 = *reinterpret_cast<const uint4*>(smem + SQ + sw128_off(rr[1], 16 * c4 + 8 * c));
                    const uint32_t kw[4] = {w.x, w.y, w.z, w.w}, qw0[4] = {q0.x, q0.y, q0.z, q0.w}, qw1[4] = {q1.x, q1.y, q1.z, q1.w};
#pragma unroll
                    for (int e = 0; e < 4; ++e) {
                        acc0 += bf16_lo(qw0[e]) * bf16_lo(kw[e]) + bf16_hi(qw0[e]) * bf16_hi(kw[e]);
                        acc1 += bf16_lo(qw1[e]) * bf16_lo(kw[e]) + bf16_hi(qw1[e]) * bf16_hi(kw[e]);
                    }
                }
            }
            acc0 += __shfl_xor_sync(0xffffffffu, acc0, 1), acc1 += __shfl_xor_sync(0xffffffffu, acc1, 1);
            acc0 += __shfl_xor_sync(0xffffffffu, acc0, 2), acc1 += __shfl_xor_sync(0xffffffffu, acc1, 2);
            s_pre[0][j] = (j < prefix && (!p.causal || j <= qtok[0])) ? acc0 : -INFINITY;
            s_pre[1][j] = (j < prefix && (!p.causal || j <= qtok[1])) ? acc1 : -INFINITY;
        }
        wgmma_wait<0>();
        fence_regs(s);
        // pass 1: row max (score s[4 jn + 2 i + c] is key 8 jn + 2 c4 + c of row i)
        float m[2], msc[2], l[2];
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            m[i] = -INFINITY;
#pragma unroll
            for (int j = 0; j < MAX_PREFIX; ++j) m[i] = fmaxf(m[i], s_pre[i][j]);
        }
#pragma unroll
        for (int jn = 0; jn < NK / 8; ++jn)
#pragma unroll
            for (int i = 0; i < 2; ++i)
#pragma unroll
                for (int c = 0; c < 2; ++c) {
                    const int key = 8 * jn + 2 * c4 + c;
                    if (key >= kmin[i] && key < kmax[i]) m[i] = fmaxf(m[i], s[4 * jn + 2 * i + c]);
                }
        float p_pre[2][MAX_PREFIX];
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            m[i] = fmaxf(m[i], __shfl_xor_sync(0xffffffffu, m[i], 1));
            m[i] = fmaxf(m[i], __shfl_xor_sync(0xffffffffu, m[i], 2));
            msc[i] = (m[i] == -INFINITY) ? 0.f : m[i] * p.scale_log2;
            l[i] = 0.f;
#pragma unroll
            for (int j = 0; j < MAX_PREFIX; ++j) {
                p_pre[i][j] = (s_pre[i][j] == -INFINITY) ? 0.f : ex2f(s_pre[i][j] * p.scale_log2 - msc[i]);
                if (c4 == 0) l[i] += p_pre[i][j];  // the prefix columns are counted once per row (quad sum below)
                p_pre[i][j] = bf16_round(p_pre[i][j]);
            }
        }
        // pass 2: p = exp2(s*scale*log2e - m*scale*log2e) in place, the bf16 numerators feed P·V from registers
#pragma unroll
        for (int jn = 0; jn < NK / 8; ++jn)
#pragma unroll
            for (int i = 0; i < 2; ++i)
#pragma unroll
                for (int c = 0; c < 2; ++c) {
                    const int key = 8 * jn + 2 * c4 + c;
                    float& v = s[4 * jn + 2 * i + c];
                    v = (key >= kmin[i] && key < kmax[i]) ? ex2f(v * p.scale_log2 - msc[i]) : 0.f;
                    l[i] += v;
                }
        mbar_wait(bar_v, 0);
        float o[32];
        {
            const uint32_t va = smem_u32(smem + SV);
            wgmma_fence();
#pragma unroll
            for (int kk = 0; kk < NK / 16; ++kk) {  // 16 keys per k-step
                const uint32_t a[4] = {pack_bf16x2(s[8 * kk], s[8 * kk + 1]), pack_bf16x2(s[8 * kk + 2], s[8 * kk + 3]),
                                       pack_bf16x2(s[8 * kk + 4], s[8 * kk + 5]), pack_bf16x2(s[8 * kk + 6], s[8 * kk + 7])};
                wgmma_m64n64_rs<1>(o, a, wgmma_desc_sw128(va + kk * 2048, 8192, 1024), kk > 0);
            }
            wgmma_commit();
            wgmma_wait<0>();
            fence_regs(o);
        }
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            l[i] += __shfl_xor_sync(0xffffffffu, l[i], 1);
            l[i] += __shfl_xor_sync(0xffffffffu, l[i], 2);
        }
        // epilogue: o[4 jn + 2 i + c] is dim 8 jn + 2 c4 + c of row i
#pragma unroll
        for (int j = 0; j < MAX_PREFIX; ++j) {
            if (j < prefix) {
                const __nv_bfloat16* vp = p.qkv + (seq_row0 + j) * 3 * D + 2 * D + h * 64 + 2 * c4;
#pragma unroll
                for (int jn = 0; jn < 8; ++jn) {
                    const uint32_t w = __ldg(reinterpret_cast<const uint32_t*>(vp + 8 * jn));
#pragma unroll
                    for (int i = 0; i < 2; ++i)
                        o[4 * jn + 2 * i] += p_pre[i][j] * bf16_lo(w), o[4 * jn + 2 * i + 1] += p_pre[i][j] * bf16_hi(w);
                }
            }
        }
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            if (!row_valid[i]) continue;
            const float inv = 1.f / l[i];
            __nv_bfloat16* op = p.out + (seq_row0 + qtok[i]) * D + h * 64 + 2 * c4;
#pragma unroll
            for (int jn = 0; jn < 8; ++jn)
                *reinterpret_cast<uint32_t*>(op + 8 * jn) = pack_bf16x2(o[4 * jn + 2 * i] * inv, o[4 * jn + 2 * i + 1] * inv);
            if (p.lse && c4 == 0) {
                if (p.pack) p.lse[((long)(b + pseq[i]) * p.H + h) * T + (rr[i] - pseq[i] * T)] = m[i] * p.scale + logf(l[i]);
                else p.lse[((long)b * p.H + h) * T + qtok[i]] = m[i] * p.scale + logf(l[i]);
            }
        }
    } else {
        setmaxnreg_dec<104>();
        if (warp != 8) return;
        if (lane == 0) {
            // ---------------- TMA
            const int row_q = (int)seq_row0 + prefix + 128 * qt;
            const int row_k = (int)seq_row0 + prefix;
            mbar_expect_tx(bar_qk, 16384 + 16384);
            tma_load_2d(smem + SQ, &tm, bar_qk, h * 64, row_q);
            tma_load_2d(smem + SK, &tm, bar_qk, D + h * 64, row_k);
            mbar_expect_tx(bar_v, 16384);
            tma_load_2d(smem + SV, &tm, bar_v, 2 * D + h * 64, row_k);
        }
        // ---------------- warp 8: prefix query rows (only the qt==0 CTA), CUDA cores over the smem K/V tiles
        if (qt == 0 && prefix > 0) {
            mbar_wait(bar_qk, 0);
            mbar_wait(bar_v, 0);
            for (int j = 0; j < prefix; ++j) {
                float qf[64];
                {
                    const uint4* qp = reinterpret_cast<const uint4*>(p.qkv + (seq_row0 + j) * 3 * D + h * 64);
#pragma unroll
                    for (int c = 0; c < 8; ++c) {
                        const uint4 w = __ldg(qp + c);
                        qf[c * 8 + 0] = bf16_lo(w.x), qf[c * 8 + 1] = bf16_hi(w.x), qf[c * 8 + 2] = bf16_lo(w.y);
                        qf[c * 8 + 3] = bf16_hi(w.y), qf[c * 8 + 4] = bf16_lo(w.z), qf[c * 8 + 5] = bf16_hi(w.z);
                        qf[c * 8 + 6] = bf16_lo(w.w), qf[c * 8 + 7] = bf16_hi(w.w);
                    }
                }
                auto dot_row = [&](const uint4* kp, bool from_smem, int row) {
                    float acc = 0.f;
#pragma unroll
                    for (int c = 0; c < 8; ++c) {
                        const uint4 w = from_smem ? *reinterpret_cast<const uint4*>(smem + SK + sw128_off(row, c * 8))
                                                  : __ldg(kp + c);
                        acc += qf[c * 8 + 0] * bf16_lo(w.x) + qf[c * 8 + 1] * bf16_hi(w.x) + qf[c * 8 + 2] * bf16_lo(w.y) +
                               qf[c * 8 + 3] * bf16_hi(w.y) + qf[c * 8 + 4] * bf16_lo(w.z) + qf[c * 8 + 5] * bf16_hi(w.z) +
                               qf[c * 8 + 6] * bf16_lo(w.w) + qf[c * 8 + 7] * bf16_hi(w.w);
                    }
                    return acc;
                };
                float sp[MAX_PREFIX], s[8];
                float m = -INFINITY;
#pragma unroll
                for (int t = 0; t < MAX_PREFIX; ++t) {
                    sp[t] = -INFINITY;
                    if (t < prefix && (!p.causal || t <= j))
                        sp[t] = dot_row(reinterpret_cast<const uint4*>(p.qkv + (seq_row0 + t) * 3 * D + D + h * 64), false, 0);
                    m = fmaxf(m, sp[t]);
                }
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    const int kk = lane + 32 * i;
                    s[i] = -INFINITY;
                    if (kk < HW && kk < kvrows && (!p.causal || prefix + kk <= j)) s[i] = dot_row(nullptr, true, kk);
                    m = fmaxf(m, s[i]);
                }
                m = warp_max(m);
                const float msc = m * p.scale_log2;
                float l = 0.f;
                __nv_bfloat16* pcls = reinterpret_cast<__nv_bfloat16*>(smem + SPCLS);
                __syncwarp();  // previous prefix row has finished reading pcls
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    const float e = (s[i] == -INFINITY) ? 0.f : ex2f(s[i] * p.scale_log2 - msc);
                    l += e;
                    pcls[lane + 32 * i] = __float2bfloat16_rn(e);  // keys beyond HW / kvrows get 0
                }
                l = warp_sum(l);
                __syncwarp();
                float a0 = 0.f, a1 = 0.f, c0 = 0.f, c1 = 0.f;
#pragma unroll
                for (int t = 0; t < MAX_PREFIX; ++t) {
                    if (t < prefix && sp[t] != -INFINITY) {
                        const float pe = ex2f(sp[t] * p.scale_log2 - msc);
                        l += pe;
                        const uint32_t w = __ldg(reinterpret_cast<const uint32_t*>(p.qkv + (seq_row0 + t) * 3 * D + 2 * D + h * 64) + lane);
                        a0 += bf16_round(pe) * bf16_lo(w), a1 += bf16_round(pe) * bf16_hi(w);
                    }
                }
                // O_cls = P V: the lane owns output dims (2 lane, 2 lane + 1); eight keys per iteration, the numerators come
                // as one broadcast 16-byte read, two independent accumulator pairs (the former per-key shuffle chain cost
                // ~16k cycles and made this warp the straggler of every qt == 0 CTA)
                const int kend = min(HW, kvrows);
                for (int k8 = 0; k8 < kend; k8 += 8) {
                    const uint4 pw = *reinterpret_cast<const uint4*>(pcls + k8);
                    const uint32_t pr[4] = {pw.x, pw.y, pw.z, pw.w};
#pragma unroll
                    for (int u = 0; u < 8; ++u) {
                        const float pk = (u & 1) ? bf16_hi(pr[u >> 1]) : bf16_lo(pr[u >> 1]);
                        const uint32_t w = *reinterpret_cast<const uint32_t*>(smem + SV + sw128_off(k8 + u, 2 * lane));
                        if (u & 1) c0 += pk * bf16_lo(w), c1 += pk * bf16_hi(w);
                        else a0 += pk * bf16_lo(w), a1 += pk * bf16_hi(w);
                    }
                }
                a0 += c0, a1 += c1;
                const float inv = 1.f / l;
                *reinterpret_cast<uint32_t*>(p.out + (seq_row0 + j) * D + h * 64 + 2 * lane) = pack_bf16x2(a0 * inv, a1 * inv);
                if (p.lse && lane == 0) p.lse[((long)b * p.H + h) * T + j] = m * p.scale + logf(l);
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------------------
// 128 < HW <= 256, not packed (the 256² step: T = 257 in the encoder, T = 256 in the decoder).  One CTA = one
// warpgroup = 64 query rows of one (head, image); thread 0 issues the TMA loads of the Q tile and all 256 K / V rows.
// The keys are two 128-key halves (wgmma m64n128, 64 score registers each):
//   S2 = Q·K2ᵀ for the row max only; S1 = Q·K1ᵀ, the row max complete, O = P1·V1; S2 again, O += P2·V2.
// One extra quarter of MMA work buys the single-pass softmax's numerators (rounded to bf16 against the whole row's
// max, as attn_fwd_kernel rounds them), so the patch rows do not depend on where in the row its max lies.
// Occupancy, so that one CTA's loads, softmax and MMAs overlap the other CTAs' on the SM:
//   registers  128 threads x 168 (launch bound 3) = 21 504; x 3 = 64 512 <= 65 536
//   smem       Q 8K + K 32K + V 32K + prefix scores 1K + barriers + 1K alignment slack = 75 840 B; + 1K reserved per
//              CTA, x 3 = 230 592 <= 233 472 (228 KB)
// -> three CTAs per SM.  The prefix query rows are spread over the CTAs of the (head, image) (row j goes to query
// tile j mod gridDim.x) and, within one, over its four warps (64 keys each, partial softmax states merged in smem), so
// none of them adds a one-warp pass over all keys to a CTA.
static constexpr int S256_THREADS = 128;
// smem: Q 8K | K 32K | V 32K | prefix scores [64 rows][MAX_PREFIX] | barriers; after the main rows the Q tile is the
// prefix query rows' scratch
static constexpr int S256_Q = 0, S256_K = 8192, S256_V = S256_K + 32768, S256_SPRE = S256_V + 32768;
static constexpr int S256_BAR = S256_SPRE + 64 * MAX_PREFIX * 4;
static constexpr int S256_SMEM = S256_BAR + 64 + 1024;  // + alignment slack

__global__ void __launch_bounds__(S256_THREADS, 3) attn_fwd_256_kernel(const __grid_constant__ CUtensorMap tm,
                                                                       const AttnDev p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + S256_BAR);
    uint64_t* bar_k1 = bars + 0;  // Q and keys 0..127 landed
    uint64_t* bar_k2 = bars + 1;  // keys 128..255 landed
    uint64_t* bar_v = bars + 2;   // V landed

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, c4 = lane & 3;
    const int qt = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
    const int D = p.D, T = p.T, prefix = p.prefix, HW = p.HW;
    const long seq_row0 = (long)b * T;
    const float sl2 = p.scale_log2;

    if (threadIdx.x == 0) {
        mbar_init(bar_k1, 1), mbar_init(bar_k2, 1), mbar_init(bar_v, 1);
        fence_barrier_init();
        // 64-row boxes; rows past HW (the next image, or zero fill past the buffer) are loaded and take no weight
        const int row_k = (int)seq_row0 + prefix;
        mbar_expect_tx(bar_k1, 8192 + 16384);
        tma_load_2d(smem + S256_Q, &tm, bar_k1, h * 64, row_k + 64 * qt);
        for (int i = 0; i < 2; ++i) tma_load_2d(smem + S256_K + i * 8192, &tm, bar_k1, D + h * 64, row_k + 64 * i);
        mbar_expect_tx(bar_k2, 16384);
        for (int i = 2; i < 4; ++i) tma_load_2d(smem + S256_K + i * 8192, &tm, bar_k2, D + h * 64, row_k + 64 * i);
        mbar_expect_tx(bar_v, 32768);
        for (int i = 0; i < 4; ++i) tma_load_2d(smem + S256_V + i * 8192, &tm, bar_v, 2 * D + h * 64, row_k + 64 * i);
    }
    __syncthreads();

    // thread quad (lane / 4) of warp w owns query rows 16 w + lane / 4 (+ 8) of the tile; keys [0, kmax) are visible
    int rr[2], qpos[2], kmax[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        rr[i] = 16 * warp + (lane >> 2) + 8 * i;
        qpos[i] = 64 * qt + rr[i];
        kmax[i] = p.causal ? min(HW, qpos[i] + 1) : HW;
    }
    const uint32_t qa = smem_u32(smem + S256_Q), ka = smem_u32(smem + S256_K), va = smem_u32(smem + S256_V);
    mbar_wait(bar_k1, 0);

    // scores against the prefix keys (CUDA cores): q rows from smem, k rows from global; the four threads of the quad
    // take 16 dims each.  Every patch query sees every prefix key, causal or not.  The row max starts at their max; the
    // scores wait in smem (registers are short here) until the max is final, as in attn_fwd_kernel.
    float* spre = reinterpret_cast<float*>(smem + S256_SPRE);
    float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
#pragma unroll
    for (int j = 0; j < MAX_PREFIX; ++j) {
        float acc0 = 0.f, acc1 = 0.f;
        if (j < prefix) {
            const uint4* kp = reinterpret_cast<const uint4*>(p.qkv + (seq_row0 + j) * 3 * D + D + h * 64 + 16 * c4);
#pragma unroll
            for (int c = 0; c < 2; ++c) {
                const uint4 w = __ldg(kp + c);
                const uint4 q0 = *reinterpret_cast<const uint4*>(smem + S256_Q + sw128_off(rr[0], 16 * c4 + 8 * c));
                const uint4 q1 = *reinterpret_cast<const uint4*>(smem + S256_Q + sw128_off(rr[1], 16 * c4 + 8 * c));
                const uint32_t kw[4] = {w.x, w.y, w.z, w.w}, qw0[4] = {q0.x, q0.y, q0.z, q0.w}, qw1[4] = {q1.x, q1.y, q1.z, q1.w};
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    acc0 += bf16_lo(qw0[e]) * bf16_lo(kw[e]) + bf16_hi(qw0[e]) * bf16_hi(kw[e]);
                    acc1 += bf16_lo(qw1[e]) * bf16_lo(kw[e]) + bf16_hi(qw1[e]) * bf16_hi(kw[e]);
                }
            }
        }
        acc0 += __shfl_xor_sync(0xffffffffu, acc0, 1), acc1 += __shfl_xor_sync(0xffffffffu, acc1, 1);
        acc0 += __shfl_xor_sync(0xffffffffu, acc0, 2), acc1 += __shfl_xor_sync(0xffffffffu, acc1, 2);
        if (j < prefix) {
            m[0] = fmaxf(m[0], acc0), m[1] = fmaxf(m[1], acc1);
            if (c4 == 0) spre[rr[0] * MAX_PREFIX + j] = acc0, spre[rr[1] * MAX_PREFIX + j] = acc1;
        }
    }
    __syncwarp();  // the quad's other lanes read spre
    // S = Q·Kᵀ over one 128-key half into s, keys >= kmax masked to -inf: score s[4 jn + 2 i + c] is key
    // 128 half + 8 jn + 2 c4 + c of row i
    auto scores = [&](float(&s)[64], int half) {
        wgmma_fence();
#pragma unroll
        for (int j = 0; j < 4; ++j)
            wgmma_m64n128_ss<0, 0>(s, wgmma_desc_sw128(qa + j * 32, 0, 1024),
                                   wgmma_desc_sw128(ka + half * 16384 + j * 32, 0, 1024), j > 0);
        wgmma_commit();
        wgmma_wait<0>();
        fence_regs(s);
#pragma unroll
        for (int i = 0; i < 2; ++i)
            if (kmax[i] - 128 * half < 128) {
#pragma unroll
                for (int jn = 0; jn < 16; ++jn)
#pragma unroll
                    for (int c = 0; c < 2; ++c)
                        if (128 * half + 8 * jn + 2 * c4 + c >= kmax[i]) s[4 * jn + 2 * i + c] = -INFINITY;
            }
    };
    auto row_max = [&](const float(&s)[64]) {
#pragma unroll
        for (int jn = 0; jn < 16; ++jn)
#pragma unroll
            for (int i = 0; i < 2; ++i) m[i] = fmaxf(m[i], fmaxf(s[4 * jn + 2 * i], s[4 * jn + 2 * i + 1]));
    };
    // The softmax takes the whole row's max before any numerator is formed, so that the bf16 numerators P·V consumes
    // are those of a single-pass softmax: half 2's scores are computed once for the max alone and again for P·V.
    // (Keeping both halves' 128 scores in registers, or issuing one half's MMAs under the other's softmax, needs more
    // than the 168 registers of a three-CTA SM and spills; the overlap comes from the other two CTAs instead.)
    float o[32], msc[2];
#pragma unroll 1
    for (int it = 0; it < 3; ++it) {  // half 2 (max only), half 1, half 2
        const int t = it == 0 ? 1 : it - 1;
        float s[64];
        if (it == 0) mbar_wait(bar_k2, 0);
        scores(s, t);
        if (it == 0) {
            row_max(s);
            continue;
        }
        if (it == 1) {
            row_max(s);
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                m[i] = fmaxf(m[i], __shfl_xor_sync(0xffffffffu, m[i], 1));
                m[i] = fmaxf(m[i], __shfl_xor_sync(0xffffffffu, m[i], 2));
                msc[i] = (m[i] == -INFINITY) ? 0.f : m[i] * sl2;
#pragma unroll
                for (int j = 0; j < MAX_PREFIX; ++j)  // the prefix columns are counted once per row (quad sum below)
                    if (j < prefix && c4 == 0) l[i] += ex2f(spre[rr[i] * MAX_PREFIX + j] * sl2 - msc[i]);
            }
        }
        uint32_t pk[32];
#pragma unroll
        for (int jn = 0; jn < 16; ++jn)
#pragma unroll
            for (int i = 0; i < 2; ++i)
#pragma unroll
                for (int c = 0; c < 2; ++c) {
                    float& v = s[4 * jn + 2 * i + c];
                    v = ex2f(v * sl2 - msc[i]);  // masked -inf -> 0
                    l[i] += v;
                }
#pragma unroll
        for (int k = 0; k < 32; ++k) pk[k] = pack_bf16x2(s[2 * k], s[2 * k + 1]);
        if (t == 0) mbar_wait(bar_v, 0);
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < 8; ++kk) {  // 16 keys per k-step
            const uint32_t a[4] = {pk[4 * kk], pk[4 * kk + 1], pk[4 * kk + 2], pk[4 * kk + 3]};
            wgmma_m64n64_rs<1>(o, a, wgmma_desc_sw128(va + t * 16384 + kk * 2048, 8192, 1024), t > 0 || kk > 0);
        }
        wgmma_commit();
        wgmma_wait<0>();
        fence_regs(o);
    }

    // epilogue: the prefix columns, then o[4 jn + 2 i + c] is dim 8 jn + 2 c4 + c of row i
#pragma unroll
    for (int j = 0; j < MAX_PREFIX; ++j) {
        if (j < prefix) {
            const __nv_bfloat16* vp = p.qkv + (seq_row0 + j) * 3 * D + 2 * D + h * 64 + 2 * c4;
            float pb[2];
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                pb[i] = bf16_round(ex2f(spre[rr[i] * MAX_PREFIX + j] * sl2 - msc[i]));
            }
#pragma unroll
            for (int jn = 0; jn < 8; ++jn) {
                const uint32_t w = __ldg(reinterpret_cast<const uint32_t*>(vp + 8 * jn));
#pragma unroll
                for (int i = 0; i < 2; ++i) o[4 * jn + 2 * i] += pb[i] * bf16_lo(w), o[4 * jn + 2 * i + 1] += pb[i] * bf16_hi(w);
            }
        }
    }
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        l[i] += __shfl_xor_sync(0xffffffffu, l[i], 1);
        l[i] += __shfl_xor_sync(0xffffffffu, l[i], 2);
        if (qpos[i] >= HW) continue;
        const float inv = 1.f / l[i];
        const long tok = seq_row0 + prefix + qpos[i];
        __nv_bfloat16* op = p.out + tok * D + h * 64 + 2 * c4;
#pragma unroll
        for (int jn = 0; jn < 8; ++jn)
            *reinterpret_cast<uint32_t*>(op + 8 * jn) = pack_bf16x2(o[4 * jn + 2 * i] * inv, o[4 * jn + 2 * i + 1] * inv);
        if (p.lse && c4 == 0) p.lse[((long)b * p.H + h) * T + prefix + qpos[i]] = m[i] * p.scale + logf(l[i]);
    }

    // ---------------- prefix query rows: warp w scores keys 64 w .. 64 w + 63 (warp 0 also the prefix keys) against
    // the smem K tile, accumulates its P·V from the smem V tile, and warp 0 merges the four partial states.  A causal
    // prefix row sees only the prefix keys up to itself.
    float* pnum = reinterpret_cast<float*>(smem + S256_Q);  // [4][64] bf16-rounded numerators
    float* po = pnum + 4 * 64;                              // [4][64] partial P·V
    float* pml = po + 4 * 64;                               // [4] partial max, [4] partial sum
    for (int j = qt; j < prefix; j += gridDim.x) {
        __syncthreads();  // every warp is done with the Q tile (its wgmma waited), or with the previous row's scratch
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
        auto dot = [&](const uint4* kp, int row) {  // kp: a global K row, else row `row` of the smem K tile
            float acc = 0.f;
#pragma unroll
            for (int c = 0; c < 8; ++c) {
                const uint4 w = kp ? __ldg(kp + c) : *reinterpret_cast<const uint4*>(smem + S256_K + sw128_off(row, c * 8));
                const uint32_t ww[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
                for (int e = 0; e < 4; ++e) acc += qf[c * 8 + 2 * e] * bf16_lo(ww[e]) + qf[c * 8 + 2 * e + 1] * bf16_hi(ww[e]);
            }
            return acc;
        };
        float sk[2], sp[MAX_PREFIX], mw = -INFINITY;
#pragma unroll
        for (int u = 0; u < 2; ++u) {
            const int k = 64 * warp + 32 * u + lane;
            sk[u] = (k < HW && !p.causal) ? dot(nullptr, k) : -INFINITY;
            mw = fmaxf(mw, sk[u]);
        }
#pragma unroll
        for (int t = 0; t < MAX_PREFIX; ++t) {
            sp[t] = -INFINITY;
            if (warp == 0 && t < prefix && (!p.causal || t <= j))
                sp[t] = dot(reinterpret_cast<const uint4*>(p.qkv + (seq_row0 + t) * 3 * D + D + h * 64), 0);
            mw = fmaxf(mw, sp[t]);
        }
        mw = warp_max(mw);
        const float mws = (mw == -INFINITY) ? 0.f : mw * sl2;  // a warp without visible keys keeps l = 0, O = 0
        float lw = 0.f;
#pragma unroll
        for (int u = 0; u < 2; ++u) {
            const float e = (sk[u] == -INFINITY) ? 0.f : ex2f(sk[u] * sl2 - mws);
            lw += e;
            pnum[64 * warp + 32 * u + lane] = bf16_round(e);
        }
        lw = warp_sum(lw);
        float a0 = 0.f, a1 = 0.f, c0 = 0.f, c1 = 0.f;  // the lane owns output dims (2 lane, 2 lane + 1)
#pragma unroll
        for (int t = 0; t < MAX_PREFIX; ++t) {
            if (sp[t] != -INFINITY) {
                const float pe = ex2f(sp[t] * sl2 - mws);
                lw += pe;
                const uint32_t w = __ldg(reinterpret_cast<const uint32_t*>(p.qkv + (seq_row0 + t) * 3 * D + 2 * D + h * 64) + lane);
                a0 += bf16_round(pe) * bf16_lo(w), a1 += bf16_round(pe) * bf16_hi(w);
            }
        }
        __syncwarp();
        const int kend = p.causal ? 0 : min(64, HW - 64 * warp);
        for (int k8 = 0; k8 < kend; k8 += 8) {  // numerators of keys >= HW are 0
            const float4 pa = *reinterpret_cast<const float4*>(pnum + 64 * warp + k8);
            const float4 pb = *reinterpret_cast<const float4*>(pnum + 64 * warp + k8 + 4);
            const float pr[8] = {pa.x, pa.y, pa.z, pa.w, pb.x, pb.y, pb.z, pb.w};
#pragma unroll
            for (int u = 0; u < 8; ++u) {
                const uint32_t w = *reinterpret_cast<const uint32_t*>(smem + S256_V + sw128_off(64 * warp + k8 + u, 2 * lane));
                if (u & 1) c0 += pr[u] * bf16_lo(w), c1 += pr[u] * bf16_hi(w);
                else a0 += pr[u] * bf16_lo(w), a1 += pr[u] * bf16_hi(w);
            }
        }
        if (lane == 0) pml[warp] = mw, pml[4 + warp] = lw;
        po[64 * warp + 2 * lane] = a0 + c0, po[64 * warp + 2 * lane + 1] = a1 + c1;
        __syncthreads();
        if (warp == 0) {
            float M = -INFINITY;
#pragma unroll
            for (int w = 0; w < 4; ++w) M = fmaxf(M, pml[w]);
            float L = 0.f, o0 = 0.f, o1 = 0.f;
#pragma unroll
            for (int w = 0; w < 4; ++w) {
                const float f = (pml[w] == -INFINITY) ? 0.f : ex2f((pml[w] - M) * sl2);
                L += f * pml[4 + w], o0 += f * po[64 * w + 2 * lane], o1 += f * po[64 * w + 2 * lane + 1];
            }
            const float inv = 1.f / L;
            *reinterpret_cast<uint32_t*>(p.out + (seq_row0 + j) * D + h * 64 + 2 * lane) = pack_bf16x2(o0 * inv, o1 * inv);
            if (p.lse && lane == 0) p.lse[((long)b * p.H + h) * T + j] = M * p.scale + logf(L);
        }
    }
}


// ------------------------------------------------------------------------------------------------------------
// fp32 attention (accuracy mode): CUDA cores, one CTA per (head, image), K/V tiles in padded smem, one warp per
// query row.  Used by the fp32-exact inference mode only (layers/attention.py:124 with fp32 q,k,v).
__global__ void attn_fwd_f32_kernel(const float* __restrict__ qkv, float* __restrict__ out, int T, int H, int causal,
                                    float scale) {
    extern __shared__ float sm[];
    const int D = H * 64, h = blockIdx.x, b = blockIdx.y;
    float* Ks = sm;                 // [T][65]
    float* Vs = Ks + (long)T * 65;  // [T][64]
    float* Ps = Vs + (long)T * 64;  // [nwarps][T]
    const float* base = qkv + (long)b * T * 3 * D;
    for (int i = threadIdx.x; i < T * 64; i += blockDim.x) {
        const int t = i >> 6, d = i & 63;
        Ks[t * 65 + d] = base[(long)t * 3 * D + D + h * 64 + d];
        Vs[t * 64 + d] = base[(long)t * 3 * D + 2 * D + h * 64 + d];
    }
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
    float* pw = Ps + (long)warp * T;
    for (int q = warp; q < T; q += nw) {
        const float* qp = base + (long)q * 3 * D + h * 64;
        float qf[64];
#pragma unroll
        for (int d = 0; d < 64; ++d) qf[d] = qp[d];
        const int kend = causal ? q + 1 : T;
        float m = -INFINITY;
        for (int k = lane; k < kend; k += 32) {
            float acc = 0.f;
#pragma unroll
            for (int d = 0; d < 64; ++d) acc += qf[d] * Ks[k * 65 + d];
            acc *= scale;
            pw[k] = acc;
            m = fmaxf(m, acc);
        }
        m = warp_max(m);
        float l = 0.f;
        for (int k = lane; k < kend; k += 32) {
            const float e = expf(pw[k] - m);
            pw[k] = e;
            l += e;
        }
        l = warp_sum(l);
        __syncwarp();
        float a0 = 0.f, a1 = 0.f;
        for (int k = 0; k < kend; ++k) {
            const float pk = pw[k];
            a0 += pk * Vs[k * 64 + lane], a1 += pk * Vs[k * 64 + 32 + lane];
        }
        float* op = out + ((long)b * T + q) * D + h * 64;
        op[lane] = a0 / l, op[32 + lane] = a1 / l;
        __syncwarp();
    }
}

}  // namespace vtp

using namespace vtp;

extern "C" int vtp_attention_fwd(const void* qkv, void* out, float* lse, int B, int T, int H, int prefix, int causal,
                                 vtp_stream_t st) {
    VTP_CHECK_ARG(qkv && out && B > 0 && T > 0 && H > 0, "attention_fwd: bad args");
    VTP_CHECK_ARG(prefix >= 0 && prefix <= MAX_PREFIX && prefix < T, "attention_fwd: prefix must be in [0,%d]", MAX_PREFIX);
    const int HW = T - prefix;
    VTP_CHECK_ARG(HW <= 256 || !causal, "attention_fwd: causal attention over %d > 256 non-prefix tokens is not supported",
                  HW);
    VTP_CHECK_ARG(B <= 65535 && H <= 65535, "attention_fwd: grid too large");
    const int D = H * 64;
    AttnDev p;
    p.qkv = (const __nv_bfloat16*)qkv, p.out = (__nv_bfloat16*)out, p.lse = lse;
    p.B = B, p.T = T, p.H = H, p.D = D, p.prefix = prefix, p.HW = HW, p.causal = causal;
    p.scale = 0.125f;
    p.scale_log2 = 0.125f * 1.4426950408889634f;
    p.pack = 0;
    if (!causal && T <= 64 && B > 1 && getenv("VTP_ATTN_NO_PACK") == nullptr) {
        // several whole sequences per 128-row tile; the prefix tokens become ordinary rows / columns
        p.pack = 128 / T;
        p.prefix = 0, p.HW = T;
    }
    const bool two_halves = p.HW > 128 && p.HW <= 256;  // attn_fwd_256_kernel: 64-row boxes
    CUtensorMap tm;
    uint64_t dims[2] = {(uint64_t)3 * D, (uint64_t)B * T}, strides[1] = {(uint64_t)3 * D * 2};
    uint32_t box[2] = {64, two_halves ? 64u : 128u};
    int rc = make_tmap_bf16(&tm, qkv, 2, dims, strides, box);
    if (rc) return rc;
    if (HW > 256) return attn_fwd_long(tm, p, (cudaStream_t)st);  // the score row no longer fits one thread quad
    static bool configured = false;
    if (!configured) {
        VTP_CUDA(cudaFuncSetAttribute(attn_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, ATT_SMEM));
        VTP_CUDA(cudaFuncSetAttribute(attn_fwd_256_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, S256_SMEM));
        // the full 228 KB carveout: three CTAs per SM
        VTP_CUDA(cudaFuncSetAttribute(attn_fwd_256_kernel, cudaFuncAttributePreferredSharedMemoryCarveout,
                                      cudaSharedmemCarveoutMaxShared));
        configured = true;
    }
    if (two_halves) {
        attn_fwd_256_kernel<<<dim3(ceil_div(HW, 64), H, B), S256_THREADS, S256_SMEM, (cudaStream_t)st>>>(tm, p);
    } else {
        dim3 grid(p.pack ? 1 : ceil_div(HW, 128), H, p.pack ? ceil_div(B, p.pack) : B);
        attn_fwd_kernel<<<grid, ATT_THREADS, ATT_SMEM, (cudaStream_t)st>>>(tm, p);
    }
    VTP_LAUNCH_CHECK();
    return VTP_OK;
}

extern "C" int vtp_attention_fwd_f32(const float* qkv, float* out, int B, int T, int H, int causal, vtp_stream_t st) {
    VTP_CHECK_ARG(qkv && out && B > 0 && T > 0 && H > 0 && B <= 65535, "attention_fwd_f32: bad args");
    const int nw = 8;
    const size_t smem = ((size_t)T * 65 + (size_t)T * 64 + (size_t)nw * T) * sizeof(float);
    if (smem > 220 * 1024) {  // K/V no longer fit shared memory: stream them
        VTP_CHECK_ARG(!causal, "attention_fwd_f32: causal attention over T=%d (beyond the smem-resident kernel) is not "
                               "supported", T);
        return attn_fwd_f32_tiled(qkv, out, B, T, H, (cudaStream_t)st);
    }
    static size_t configured = 0;
    if (smem > configured) {
        VTP_CUDA(cudaFuncSetAttribute(attn_fwd_f32_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        configured = smem;
    }
    attn_fwd_f32_kernel<<<dim3(H, B), nw * 32, smem, (cudaStream_t)st>>>(qkv, out, T, H, causal, 0.125f);
    VTP_LAUNCH_CHECK();
    return VTP_OK;
}
