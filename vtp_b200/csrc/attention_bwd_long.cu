// vtp_b200 — non-causal self-attention BACKWARD for any sequence length (T = prefix + HW, prefix <= 1, HW >= 1):
// training on images above 256x256.
//
// Same op and same bf16 rounding points as attn_bwd_kernel (attention_bwd.cu), whose whole sequence has to fit one CTA:
//   P = exp(s·QKᵀ − lse)      dV = Pᵀ dO      dP = dO Vᵀ      dS = s · P ∘ (dP − δ),  δ_i = Σ_d dO_id O_id
//   dQ = dS K                 dK = dSᵀ Q      then RoPEᵀ on dQ, dK
// P and dS are rounded to bf16 where they enter a patch-key GEMM; the prefix (cls) row and column stay fp32 on CUDA cores.
//
// Four launches, no atomics, every element of dqkv written once by one thread (repeat launches are bit-identical):
//   attn_bwd_delta_kernel      δ for every token into a caller-provided fp32 workspace laid out like lse
//   attn_bwd_long_dq_kernel    CTA = (128 patch queries, head, image) as attn_fwd_long_kernel: Q and dO loaded once, K and
//                              V streamed through an mbarrier ring.  Per 64-key half: S = QKᵀ and dP = dO·Vᵀ (wgmma, K-major),
//                              dS in registers, dQ += dS·K with dS as the register A operand (K consumed MN-major).  The cls
//                              key column (ds_i0 · k_0) is folded in on CUDA cores.
//   attn_bwd_long_dkdv_kernel  CTA = (128 patch keys, head, image), 64 keys per warpgroup: K and V loaded once, Q and dO
//                              streamed with that tile's lse and δ.  Everything transposed so that P and dS stay in registers
//                              as A operands: Sᵀ = K·Qᵀ, dPᵀ = V·dOᵀ, dV += Pᵀ·dO, dK += dSᵀ·Q (dO, Q MN-major).  The cls
//                              query row adds p_0j · dO_0 and ds_0j · q_0 to every patch key on CUDA cores.
//   attn_bwd_prefix_kernel     (prefix 1) one CTA per (head, image): dQ_0 over all T keys, dK_0 and dV_0 as column sums over
//                              all T queries; 8 warps take interleaved 32-token chunks and merge in a fixed order.
// S and dP are computed twice (dq and dkdv kernels): 7 patch GEMMs instead of the single-pass kernel's 5, the price of
// having no fp32 atomics on dQ.
#include "attention_bwd.cuh"
#include "host.h"
#include "ptx.cuh"

namespace vtp {

namespace {

constexpr int BL_THREADS = 384;  // 2 consumer warpgroups + warpgroup 2 (warp 8: producer)
constexpr int BL_NSTAGE = 2;
constexpr int BL_TILE = 128 * 128;  // 128 rows x 64 bf16, 128B-swizzled
// dq kernel: Q | dO | NSTAGE x (K | V) | barriers
constexpr int DQ_Q = 0, DQ_DO = BL_TILE, DQ_KV = 2 * BL_TILE, DQ_BAR = DQ_KV + BL_NSTAGE * 2 * BL_TILE;
constexpr int DQ_SMEM = DQ_BAR + 128 + 1024;  // + alignment slack
// dkdv kernel: K | V | NSTAGE x (Q | dO) | NSTAGE x (lse·log2e [128] | δ [128]) | barriers
constexpr int KV_K = 0, KV_V = BL_TILE, KV_QD = 2 * BL_TILE, KV_LD = KV_QD + BL_NSTAGE * 2 * BL_TILE;
constexpr int KV_BAR = KV_LD + BL_NSTAGE * 1024;
constexpr int KV_SMEM = KV_BAR + 128 + 1024;

struct AttnBwdLongDev {
    const __nv_bfloat16* qkv;   // [B*T][3D] post-RoPE q,k ; v
    const __nv_bfloat16* o;     // [B*T][D]
    const __nv_bfloat16* dout;  // [B*T][D]
    const float* lse;           // [B][H][T]
    float* delta;               // [B][H][T] workspace: δ = Σ dO·O
    __nv_bfloat16* dqkv;        // [B*T][3D] gradient w.r.t. the PRE-RoPE qkv
    const __nv_bfloat16* rope_sin;  // [HW][64] or null
    const __nv_bfloat16* rope_cos;
    int B, T, H, D, prefix, HW;
    float scale, scale_log2;
};

// 8 threads per (token, head), each one 16-byte chunk of the 64 dims, summed over the 8 lanes
__global__ void __launch_bounds__(256) attn_bwd_delta_kernel(const AttnBwdLongDev p) {
    const long gid = (long)blockIdx.x * blockDim.x + threadIdx.x;
    const long pair = gid >> 3;  // token * H + head
    const int c = (int)(gid & 7);
    const bool valid = pair < (long)p.B * p.T * p.H;
    float acc = 0.f;
    if (valid) {
        const long tok = pair / p.H;
        const int h = (int)(pair - tok * p.H);
        const uint4 a = __ldg(reinterpret_cast<const uint4*>(p.dout + tok * p.D + h * 64) + c);
        const uint4 w = __ldg(reinterpret_cast<const uint4*>(p.o + tok * p.D + h * 64) + c);
        const uint32_t aw[4] = {a.x, a.y, a.z, a.w}, ww[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
        for (int e = 0; e < 4; ++e) acc += bf16_lo(aw[e]) * bf16_lo(ww[e]) + bf16_hi(aw[e]) * bf16_hi(ww[e]);
    }
    acc += __shfl_xor_sync(0xffffffffu, acc, 1);
    acc += __shfl_xor_sync(0xffffffffu, acc, 2);
    acc += __shfl_xor_sync(0xffffffffu, acc, 4);
    if (valid && c == 0) {
        const long tok = pair / p.H;
        const int h = (int)(pair - tok * p.H);
        const long b = tok / p.T;
        p.delta[(b * p.H + h) * p.T + (tok - b * p.T)] = acc;
    }
}

__global__ void __launch_bounds__(BL_THREADS, 1) attn_bwd_long_dq_kernel(const __grid_constant__ CUtensorMap tm_qkv,
                                                                          const __grid_constant__ CUtensorMap tm_do,
                                                                          const AttnBwdLongDev p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + DQ_BAR);
    uint64_t* bar_q = bars;               // Q and dO landed
    uint64_t* full = bars + 1;            // [NSTAGE] K and V landed
    uint64_t* empty = full + BL_NSTAGE;   // [NSTAGE] released by the 8 consumer warps

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int qt = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
    const int D = p.D, T = p.T, prefix = p.prefix, HW = p.HW;
    const long row0 = (long)b * T;
    const int nkt = (HW + 127) / 128;

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tm_qkv);
        tma_prefetch_desc(&tm_do);
        mbar_init(bar_q, 1);
        for (int s = 0; s < BL_NSTAGE; ++s) mbar_init(full + s, 1), mbar_init(empty + s, 8);
        fence_barrier_init();
    }
    __syncthreads();

    if (warp < 8) {
        setmaxnreg_inc<200>();
        const int wg = warp >> 2, tw = threadIdx.x & 127, c4 = lane & 3;
        int rr[2], qi[2];
        bool qvalid[2];
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            rr[i] = 64 * wg + 16 * (tw >> 5) + (lane >> 2) + 8 * i;
            qi[i] = 128 * qt + rr[i];
            qvalid[i] = qi[i] < HW;  // rows >= HW: the next image's rows or TMA zero fill
        }
        const __nv_bfloat16* kcls = p.qkv + row0 * 3 * D + D + h * 64;
        const __nv_bfloat16* vcls = p.qkv + row0 * 3 * D + 2 * D + h * 64;
        mbar_wait(bar_q, 0);
        // per-row scalars: lse·log2e, δ, and the cls-key column ds_i0 (fp32, CUDA cores)
        float lsc[2], dl[2], ds_cls[2];
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            const long li = ((long)b * p.H + h) * T + prefix + qi[i];
            lsc[i] = qvalid[i] ? p.lse[li] * LOG2E : 0.f;
            dl[i] = qvalid[i] ? p.delta[li] : 0.f;
            ds_cls[i] = 0.f;
            if (prefix > 0) {
                const float s0 = quad_dot(smem + DQ_Q, rr[i], kcls, c4);
                const float dp0 = quad_dot(smem + DQ_DO, rr[i], vcls, c4);
                if (qvalid[i]) ds_cls[i] = p.scale * ex2f(s0 * p.scale_log2 - lsc[i]) * (dp0 - dl[i]);
            }
        }
        float dq[32];
#pragma unroll
        for (int k = 0; k < 32; ++k) dq[k] = 0.f;
        const uint32_t aQ = smem_u32(smem + DQ_Q) + wg * 8192, aDO = smem_u32(smem + DQ_DO) + wg * 8192;
        for (int t = 0; t < nkt; ++t) {
            const int st = t % BL_NSTAGE;
            mbar_wait(full + st, (t / BL_NSTAGE) & 1);
            const uint32_t aK = smem_u32(smem + DQ_KV + st * 2 * BL_TILE), aV = aK + BL_TILE;
            const int klim = HW - 128 * t;  // keys >= klim of this tile take no weight
#pragma unroll 1
            for (int half = 0; half < 2 && 64 * half < klim; ++half) {
                float s[32], dp[32];
                wgmma_fence();
#pragma unroll
                for (int j = 0; j < 4; ++j)
                    wgmma_m64n64_ss<0, 0>(s, wgmma_desc_sw128(aQ + j * 32, 0, 1024),
                                          wgmma_desc_sw128(aK + half * 8192 + j * 32, 0, 1024), j > 0);
#pragma unroll
                for (int j = 0; j < 4; ++j)
                    wgmma_m64n64_ss<0, 0>(dp, wgmma_desc_sw128(aDO + j * 32, 0, 1024),
                                          wgmma_desc_sw128(aV + half * 8192 + j * 32, 0, 1024), j > 0);
                wgmma_commit();
                wgmma_wait<0>();
                fence_regs(s);
                fence_regs(dp);
#pragma unroll
                for (int jn = 0; jn < 8; ++jn)
#pragma unroll
                    for (int i = 0; i < 2; ++i)
#pragma unroll
                        for (int c = 0; c < 2; ++c) {
                            const int e = 4 * jn + 2 * i + c;
                            float de = 0.f;
                            if (qvalid[i] && 64 * half + 8 * jn + 2 * c4 + c < klim) {
                                const float pe = ex2f(s[e] * p.scale_log2 - lsc[i]);
                                de = p.scale * pe * (dp[e] - dl[i]);
                            }
                            s[e] = de;
                        }
                uint32_t a[4][4];
                pack_a(s, a);
                wgmma_fence();
#pragma unroll
                for (int kk = 0; kk < 4; ++kk)  // 16 keys per k-step, K as the MN-major B operand
                    wgmma_m64n64_rs<1>(dq, a[kk], wgmma_desc_sw128(aK + (4 * half + kk) * 2048, 8192, 1024), 1);
                wgmma_commit();
                wgmma_wait<0>();
                fence_regs(dq);
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(empty + st);
        }
        // epilogue: rows >= HW are not stored
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            if (!qvalid[i]) continue;
            const bool rope = p.rope_sin != nullptr;
            store_grad_row(dq, i, ds_cls[i], prefix > 0 ? kcls : nullptr, rope ? p.rope_sin + (long)qi[i] * 64 : nullptr,
                           rope ? p.rope_cos + (long)qi[i] * 64 : nullptr,
                           p.dqkv + (row0 + prefix + qi[i]) * 3 * D + h * 64, c4);
        }
    } else {
        setmaxnreg_dec<104>();
        if (warp != 8 || lane != 0) return;
        // ---------------- TMA producer
        const int row_k = (int)row0 + prefix;
        mbar_expect_tx(bar_q, 2 * BL_TILE);
        tma_load_2d(smem + DQ_Q, &tm_qkv, bar_q, h * 64, row_k + 128 * qt);
        tma_load_2d(smem + DQ_DO, &tm_do, bar_q, h * 64, row_k + 128 * qt);
        for (int t = 0; t < nkt; ++t) {
            const int st = t % BL_NSTAGE;
            if (t >= BL_NSTAGE) mbar_wait(empty + st, ((t / BL_NSTAGE) - 1) & 1);
            uint8_t* kv = smem + DQ_KV + st * 2 * BL_TILE;
            mbar_expect_tx(full + st, 2 * BL_TILE);
            tma_load_2d(kv, &tm_qkv, full + st, D + h * 64, row_k + 128 * t);
            tma_load_2d(kv + BL_TILE, &tm_qkv, full + st, 2 * D + h * 64, row_k + 128 * t);
        }
    }
}

__global__ void __launch_bounds__(BL_THREADS, 1) attn_bwd_long_dkdv_kernel(const __grid_constant__ CUtensorMap tm_qkv,
                                                                            const __grid_constant__ CUtensorMap tm_do,
                                                                            const AttnBwdLongDev p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + KV_BAR);
    uint64_t* bar_kv = bars;              // K and V landed
    uint64_t* full = bars + 1;            // [NSTAGE] Q, dO (TMA) and lse, δ (32 producer lanes) landed
    uint64_t* empty = full + BL_NSTAGE;   // [NSTAGE] released by the 8 consumer warps

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int kt = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
    const int D = p.D, T = p.T, prefix = p.prefix, HW = p.HW;
    const long row0 = (long)b * T;
    const int nqt = (HW + 127) / 128;
    const long lrow = ((long)b * p.H + h) * T;  // lse / δ row of this (image, head)

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tm_qkv);
        tma_prefetch_desc(&tm_do);
        mbar_init(bar_kv, 1);
        for (int s = 0; s < BL_NSTAGE; ++s) mbar_init(full + s, 1 + 32), mbar_init(empty + s, 8);
        fence_barrier_init();
    }
    __syncthreads();

    if (warp < 8) {
        setmaxnreg_inc<200>();
        const int wg = warp >> 2, tw = threadIdx.x & 127, c4 = lane & 3;
        int rr[2], kj[2];
        bool kvalid[2];
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            rr[i] = 64 * wg + 16 * (tw >> 5) + (lane >> 2) + 8 * i;
            kj[i] = 128 * kt + rr[i];
            kvalid[i] = kj[i] < HW;
        }
        const __nv_bfloat16* qcls = p.qkv + row0 * 3 * D + h * 64;  // q of the cls query
        const __nv_bfloat16* docls = p.dout + row0 * D + h * 64;     // dO of the cls query
        mbar_wait(bar_kv, 0);
        // the cls query row against my keys: p_0j, ds_0j (fp32, CUDA cores)
        float p0j[2] = {0.f, 0.f}, ds0j[2] = {0.f, 0.f};
        if (prefix > 0) {
            const float lse0 = p.lse[lrow] * LOG2E, dl0 = p.delta[lrow];
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                const float s = quad_dot(smem + KV_K, rr[i], qcls, c4);
                const float dp = quad_dot(smem + KV_V, rr[i], docls, c4);
                if (kvalid[i]) {
                    p0j[i] = ex2f(s * p.scale_log2 - lse0);
                    ds0j[i] = p.scale * p0j[i] * (dp - dl0);
                }
            }
        }
        float dk[32], dv[32];
#pragma unroll
        for (int k = 0; k < 32; ++k) dk[k] = 0.f, dv[k] = 0.f;
        const uint32_t aK = smem_u32(smem + KV_K) + wg * 8192, aV = smem_u32(smem + KV_V) + wg * 8192;
        for (int t = 0; t < nqt; ++t) {
            const int st = t % BL_NSTAGE;
            mbar_wait(full + st, (t / BL_NSTAGE) & 1);
            const uint32_t aQ = smem_u32(smem + KV_QD + st * 2 * BL_TILE), aDO = aQ + BL_TILE;
            const float* lse_s = reinterpret_cast<const float*>(smem + KV_LD + st * 1024);
            const float* dl_s = lse_s + 128;
            const int qlim = HW - 128 * t;  // query columns >= qlim of this tile take no weight
#pragma unroll 1
            for (int half = 0; half < 2 && 64 * half < qlim; ++half) {
                float s[32], dp[32];  // Sᵀ, dPᵀ: rows = my keys, columns = 64 queries
                wgmma_fence();
#pragma unroll
                for (int j = 0; j < 4; ++j)
                    wgmma_m64n64_ss<0, 0>(s, wgmma_desc_sw128(aK + j * 32, 0, 1024),
                                          wgmma_desc_sw128(aQ + half * 8192 + j * 32, 0, 1024), j > 0);
#pragma unroll
                for (int j = 0; j < 4; ++j)
                    wgmma_m64n64_ss<0, 0>(dp, wgmma_desc_sw128(aV + j * 32, 0, 1024),
                                          wgmma_desc_sw128(aDO + half * 8192 + j * 32, 0, 1024), j > 0);
                wgmma_commit();
                wgmma_wait<0>();
                fence_regs(s);
                fence_regs(dp);
#pragma unroll
                for (int jn = 0; jn < 8; ++jn)
#pragma unroll
                    for (int c = 0; c < 2; ++c) {
                        const int qc = 64 * half + 8 * jn + 2 * c4 + c;
                        const float lq = lse_s[qc], dq = dl_s[qc];
#pragma unroll
                        for (int i = 0; i < 2; ++i) {
                            const int e = 4 * jn + 2 * i + c;
                            float pe = 0.f, de = 0.f;
                            if (kvalid[i] && qc < qlim) {
                                pe = ex2f(s[e] * p.scale_log2 - lq);
                                de = p.scale * pe * (dp[e] - dq);
                            }
                            s[e] = pe, dp[e] = de;
                        }
                    }
                uint32_t ap[4][4], as[4][4];
                pack_a(s, ap);
                pack_a(dp, as);
                wgmma_fence();
#pragma unroll
                for (int kk = 0; kk < 4; ++kk) {  // 16 queries per k-step, dO and Q as MN-major B operands
                    wgmma_m64n64_rs<1>(dv, ap[kk], wgmma_desc_sw128(aDO + (4 * half + kk) * 2048, 8192, 1024), 1);
                    wgmma_m64n64_rs<1>(dk, as[kk], wgmma_desc_sw128(aQ + (4 * half + kk) * 2048, 8192, 1024), 1);
                }
                wgmma_commit();
                wgmma_wait<0>();
                fence_regs(dv);
                fence_regs(dk);
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(empty + st);
        }
        // epilogue: my key rows kj; rows >= HW are not stored
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            if (!kvalid[i]) continue;
            const bool rope = p.rope_sin != nullptr;
            __nv_bfloat16* drow = p.dqkv + (row0 + prefix + kj[i]) * 3 * D + h * 64;
            store_grad_row(dv, i, p0j[i], prefix > 0 ? docls : nullptr, nullptr, nullptr, drow + 2 * D, c4);
            store_grad_row(dk, i, ds0j[i], prefix > 0 ? qcls : nullptr, rope ? p.rope_sin + (long)kj[i] * 64 : nullptr,
                           rope ? p.rope_cos + (long)kj[i] * 64 : nullptr, drow + D, c4);
        }
    } else {
        setmaxnreg_dec<104>();
        if (warp != 8) return;
        // ---------------- producer warp: lane 0 issues the TMA loads, all 32 lanes stage lse·log2e and δ
        const int row_k = (int)row0 + prefix;
        if (lane == 0) {
            mbar_expect_tx(bar_kv, 2 * BL_TILE);
            tma_load_2d(smem + KV_K, &tm_qkv, bar_kv, D + h * 64, row_k + 128 * kt);
            tma_load_2d(smem + KV_V, &tm_qkv, bar_kv, 2 * D + h * 64, row_k + 128 * kt);
        }
        for (int t = 0; t < nqt; ++t) {
            const int st = t % BL_NSTAGE;
            if (t >= BL_NSTAGE) mbar_wait(empty + st, ((t / BL_NSTAGE) - 1) & 1);
            if (lane == 0) {
                uint8_t* qd = smem + KV_QD + st * 2 * BL_TILE;
                mbar_expect_tx(full + st, 2 * BL_TILE);
                tma_load_2d(qd, &tm_qkv, full + st, h * 64, row_k + 128 * t);
                tma_load_2d(qd + BL_TILE, &tm_do, full + st, h * 64, row_k + 128 * t);
            }
            float* lse_s = reinterpret_cast<float*>(smem + KV_LD + st * 1024);
#pragma unroll
            for (int r = lane; r < 128; r += 32) {
                const int q = 128 * t + r;
                lse_s[r] = q < HW ? p.lse[lrow + prefix + q] * LOG2E : 0.f;
                lse_s[128 + r] = q < HW ? p.delta[lrow + prefix + q] : 0.f;
            }
            mbar_arrive(full + st);
        }
    }
}

// Prefix (cls) token, prefix == 1: dQ_0 = Σ_t ds_0t k_t, dK_0 = Σ_t ds_t0 q_t, dV_0 = Σ_t p_t0 dO_t over all T tokens (t = 0
// included), fp32 throughout.  Warp w takes the 32-token chunks 32 w + 256 n; a lane scores its token (four 64-dim dot
// products against the cls vectors, broadcast from shared memory), then the warp accumulates with the lane owning dims
// (2 lane, 2 lane + 1); warp 0 sums the 8 partials in warp order.
constexpr int PB_WARPS = 8;

__global__ void __launch_bounds__(PB_WARPS * 32) attn_bwd_prefix_kernel(const AttnBwdLongDev p) {
    __shared__ float cls[4][64];  // q_0, k_0, v_0, dO_0
    __shared__ float part[PB_WARPS][3][64];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int h = blockIdx.x % p.H, b = blockIdx.x / p.H;
    const int D = p.D, T = p.T;
    const long row0 = (long)b * T, lrow = ((long)b * p.H + h) * T;
    const long rs = 3L * D;  // qkv row stride (elements)
    if (threadIdx.x < 256) {
        const int v = threadIdx.x >> 6, d = threadIdx.x & 63;
        const __nv_bfloat16* src = v < 3 ? p.qkv + row0 * rs + v * D + h * 64 : p.dout + row0 * D + h * 64;
        cls[v][d] = __bfloat162float(src[d]);
    }
    __syncthreads();
    const float lse0 = p.lse[lrow] * LOG2E, dl0 = p.delta[lrow];
    float aq0 = 0.f, aq1 = 0.f, ak0 = 0.f, ak1 = 0.f, av0 = 0.f, av1 = 0.f;
    for (int k0 = 32 * warp; k0 < T; k0 += 32 * PB_WARPS) {
        const int t = k0 + lane;
        float ds_0t = 0.f, ds_t0 = 0.f, p_t0 = 0.f;
        if (t < T) {
            const uint4* qp = reinterpret_cast<const uint4*>(p.qkv + (row0 + t) * rs + h * 64);
            const uint4* kp = reinterpret_cast<const uint4*>(p.qkv + (row0 + t) * rs + D + h * 64);
            const uint4* vp = reinterpret_cast<const uint4*>(p.qkv + (row0 + t) * rs + 2 * D + h * 64);
            const uint4* dp = reinterpret_cast<const uint4*>(p.dout + (row0 + t) * D + h * 64);
            float s0t = 0.f, dp0t = 0.f, st0 = 0.f, dpt0 = 0.f;
#pragma unroll
            for (int c = 0; c < 8; ++c) {
                const uint4 wq = __ldg(qp + c), wk = __ldg(kp + c), wv = __ldg(vp + c), wd = __ldg(dp + c);
                const uint32_t q4[4] = {wq.x, wq.y, wq.z, wq.w}, k4[4] = {wk.x, wk.y, wk.z, wk.w};
                const uint32_t v4[4] = {wv.x, wv.y, wv.z, wv.w}, d4[4] = {wd.x, wd.y, wd.z, wd.w};
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const int d = 8 * c + 2 * e;
                    s0t += cls[0][d] * bf16_lo(k4[e]) + cls[0][d + 1] * bf16_hi(k4[e]);
                    dp0t += cls[3][d] * bf16_lo(v4[e]) + cls[3][d + 1] * bf16_hi(v4[e]);
                    st0 += bf16_lo(q4[e]) * cls[1][d] + bf16_hi(q4[e]) * cls[1][d + 1];
                    dpt0 += bf16_lo(d4[e]) * cls[2][d] + bf16_hi(d4[e]) * cls[2][d + 1];
                }
            }
            const float p_0t = ex2f(s0t * p.scale_log2 - lse0);
            ds_0t = p.scale * p_0t * (dp0t - dl0);
            p_t0 = ex2f(st0 * p.scale_log2 - p.lse[lrow + t] * LOG2E);
            ds_t0 = p.scale * p_t0 * (dpt0 - p.delta[lrow + t]);
        }
        const int n = min(32, T - k0);
        for (int u = 0; u < n; ++u) {
            const float a = __shfl_sync(0xffffffffu, ds_0t, u), bb = __shfl_sync(0xffffffffu, ds_t0, u);
            const float c = __shfl_sync(0xffffffffu, p_t0, u);
            const long r = row0 + k0 + u;
            const uint32_t wk = __ldg(reinterpret_cast<const uint32_t*>(p.qkv + r * rs + D + h * 64) + lane);
            const uint32_t wq = __ldg(reinterpret_cast<const uint32_t*>(p.qkv + r * rs + h * 64) + lane);
            const uint32_t wd = __ldg(reinterpret_cast<const uint32_t*>(p.dout + r * D + h * 64) + lane);
            aq0 += a * bf16_lo(wk), aq1 += a * bf16_hi(wk);
            ak0 += bb * bf16_lo(wq), ak1 += bb * bf16_hi(wq);
            av0 += c * bf16_lo(wd), av1 += c * bf16_hi(wd);
        }
    }
    part[warp][0][2 * lane] = aq0, part[warp][0][2 * lane + 1] = aq1;
    part[warp][1][2 * lane] = ak0, part[warp][1][2 * lane + 1] = ak1;
    part[warp][2][2 * lane] = av0, part[warp][2][2 * lane + 1] = av1;
    __syncthreads();
    if (warp != 0) return;
#pragma unroll
    for (int v = 0; v < 3; ++v) {
        float x0 = 0.f, x1 = 0.f;
#pragma unroll
        for (int w = 0; w < PB_WARPS; ++w) x0 += part[w][v][2 * lane], x1 += part[w][v][2 * lane + 1];
        *reinterpret_cast<uint32_t*>(p.dqkv + row0 * rs + v * D + h * 64 + 2 * lane) = pack_bf16x2(x0, x1);
    }
}

}  // namespace

}  // namespace vtp

using namespace vtp;

extern "C" int vtp_attention_bwd_long(const void* qkv, const void* o, const void* dout, const float* lse, float* delta_ws,
                                      void* dqkv, const void* rope_sin, const void* rope_cos, int B, int T, int H,
                                      int prefix, vtp_stream_t stream) {
    VTP_CHECK_ARG(qkv && o && dout && lse && delta_ws && dqkv && B > 0 && T > 0 && H > 0, "attention_bwd_long: bad args");
    VTP_CHECK_ARG(prefix == 0 || prefix == 1, "attention_bwd_long: prefix must be 0 or 1");
    VTP_CHECK_ARG((rope_sin == nullptr) == (rope_cos == nullptr), "attention_bwd_long: rope tables");
    const int HW = T - prefix;
    VTP_CHECK_ARG(HW >= 1, "attention_bwd_long: no non-prefix tokens");
    VTP_CHECK_ARG(B <= 65535 && H <= 65535 && (long)B * T <= 0x7fffffffL && (long)B * H <= 0x7fffffffL &&
                      (long)B * T * H * 8 / 256 < 0x7fffffffL,
                  "attention_bwd_long: grid too large");
    const int D = H * 64;
    AttnBwdLongDev p;
    p.qkv = (const __nv_bfloat16*)qkv, p.o = (const __nv_bfloat16*)o, p.dout = (const __nv_bfloat16*)dout;
    p.lse = lse, p.delta = delta_ws, p.dqkv = (__nv_bfloat16*)dqkv;
    p.rope_sin = (const __nv_bfloat16*)rope_sin, p.rope_cos = (const __nv_bfloat16*)rope_cos;
    p.B = B, p.T = T, p.H = H, p.D = D, p.prefix = prefix, p.HW = HW;
    p.scale = 0.125f, p.scale_log2 = 0.125f * 1.4426950408889634f;
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
        VTP_CUDA(cudaFuncSetAttribute(attn_bwd_long_dq_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, DQ_SMEM));
        VTP_CUDA(cudaFuncSetAttribute(attn_bwd_long_dkdv_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, KV_SMEM));
        configured = true;
    }
    const cudaStream_t st = (cudaStream_t)stream;
    const long pairs = (long)B * T * H;
    attn_bwd_delta_kernel<<<(unsigned)((pairs * 8 + 255) / 256), 256, 0, st>>>(p);
    VTP_LAUNCH_CHECK();
    const dim3 grid(ceil_div(HW, 128), H, B);
    attn_bwd_long_dq_kernel<<<grid, BL_THREADS, DQ_SMEM, st>>>(tq, td, p);
    VTP_LAUNCH_CHECK();
    attn_bwd_long_dkdv_kernel<<<grid, BL_THREADS, KV_SMEM, st>>>(tq, td, p);
    VTP_LAUNCH_CHECK();
    if (prefix > 0) {
        attn_bwd_prefix_kernel<<<B * H, PB_WARPS * 32, 0, st>>>(p);
        VTP_LAUNCH_CHECK();
    }
    return VTP_OK;
}
