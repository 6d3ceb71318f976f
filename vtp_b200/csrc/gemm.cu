// vtp_b200 — persistent, warp-specialised wgmma GEMM for sm_90a.
//
//   out[M,N] = epilogue( A[M,K] · B[N,K]ᵀ )      bf16 operands, fp32 accumulators
//
// Roles (512 threads): warpgroup 0 = TMA producer (one thread), warpgroups 1 and 2 = MMA consumers, warpgroup 3 =
// epilogue.  BM = 128 (each consumer warpgroup issues m64 wgmma for its 64 rows), BN in {64, 128}, BK = 64 bf16 = one 128B
// swizzle span, a STAGES-deep TMA / mbarrier ring.  Operands may be K-major or MN-major (wgmma transpose bits), so forward
// (NT), dgrad (NN) and wgrad (TN) all run through this one kernel; wgrad uses split-K + fp32 atomics.  After the mainloop
// the consumers dump their accumulators into an fp32 tile in shared memory and go straight on to the next tile; the four
// epilogue warps run the epilogue from that tile with one output row per lane (32-row slabs).  Two mbarriers hand the
// tile over (acc_full: dumped, acc_empty: read), so the epilogue of tile t runs under the mainloop of tile t+1.
//
// Fused epilogues (all optional): +bias, bf16 rounding point, GELU, SwiGLU gate (8-interleaved w1|w2), axial
// RoPE on q/k (bf16 arithmetic exactly as layers/attention.py:12-23,70-89), +residual, row remap (cls-token
// slot), PixelShuffle NCHW store, secondary pre-activation output.
#include <stdlib.h>

#include "host.h"
#include "ptx.cuh"

namespace vtp {

static constexpr int BM = 128;
static constexpr int BK = 64;
static constexpr int A_BYTES = BM * BK * 2;
static constexpr int NUM_THREADS = 512;  // producer warpgroup + 2 MMA consumer warpgroups + 1 epilogue warpgroup
static constexpr int NUM_MMA_WARPS = 8;

struct GemmDev {
    int M, N, K;
    int a_mn, b_mn;
    int num_m_blocks, num_n_blocks, num_k_blocks, kb_per_split, num_splits;
    void* out;
    int ldo, out_dtype;
    const float* bias;
    int act, round_bf16;
    const void* resid;
    int ldr, resid_dtype;
    int accumulate;
    int rr_group, rr_skip;
    const __nv_bfloat16* rope_sin;
    const __nv_bfloat16* rope_cos;
    int rope_tokens, rope_prefix, rope_cols;
    int ps_r, ps_gh, ps_gw, ps_cout;
    __nv_bfloat16* out2;
    int ldo2;
    // implicit 3x3 / pad-1 convolution over an NHWC activation (A operand loaded by 4-D TMA, zero fill = padding)
    int conv_C, conv_H, conv_W, conv_TW, conv_TH, conv_tiles_h, conv_tiles_w, conv_B;
    const __nv_bfloat16* mask_pos;  // optional: out *= (mask_pos[row][col] > 0)   (ReLU backward in the dgrad epilogue)
    int ldm;
};

__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752f)); }

// ---------------------------------------------------------------------------------------------------- epilogue
// 4 epilogue warps.  Warp q owns row quarter q of the tile and all of its 64-column units.  A unit is processed in two
// phases:
//   A (row owner: lane = output row)  accumulator tile -> registers, +bias, rounding point, activation / RoPE
//   B (cooperative)  the slab goes, 32 columns at a time, through a per-warp XOR-swizzled fp32 staging tile (4 KB) so
//     that every global access is a contiguous 128-byte line per quarter-warp: residual read (prefetched into registers
//     before the accumulator is even waited for), dtype conversion, store / red.add / PixelShuffle scatter.
static constexpr int STG_FLOATS = 32 * 32;  // per epilogue warp
static constexpr int NUM_EPI_WARPS = 4;

__device__ __forceinline__ int stg_off(int r, int chunk /*0..7*/) { return r * 32 + ((chunk ^ (r & 7)) << 2); }

__device__ __forceinline__ long out_row(const GemmDev& p, int grow) {
    if (p.conv_C) {  // grow = m_blk * 128 + r : tile (b, ty, tx), pixel r of a conv_TH x conv_TW patch
        const int m_blk = grow >> 7, r = grow & 127;
        const int tx = m_blk % p.conv_tiles_w, ty = (m_blk / p.conv_tiles_w) % p.conv_tiles_h;
        const int b = m_blk / (p.conv_tiles_w * p.conv_tiles_h);
        const int h = ty * p.conv_TH + r / p.conv_TW, w = tx * p.conv_TW + r % p.conv_TW;
        return (h < p.conv_H && w < p.conv_W && b < p.conv_B) ? ((long)b * p.conv_H + h) * p.conv_W + w : -1;
    }
    if (grow >= p.M) return -1;
    if (p.rr_group <= 0) return grow;
    if (p.rr_skip >= 0)  // expansion: leave rr_skip rows free in front of every group (cls slot)
        return (long)(grow / p.rr_group) * (p.rr_group + p.rr_skip) + p.rr_skip + grow % p.rr_group;
    const int tok = grow % p.rr_group;  // compaction: drop the first -rr_skip rows of every group
    return tok < -p.rr_skip ? -1 : (long)(grow / p.rr_group) * (p.rr_group + p.rr_skip) + tok + p.rr_skip;
}

// warm the residual lines of one unit in L2 (no registers held): row 4*it + lane/8, one 128-byte line per 8 lanes
__device__ __forceinline__ void prefetch_resid_l2(const GemmDev& p, int lane, const long (&orow8)[8], int ocol0, int ncols,
                                                  int Nout) {
    if ((lane & 7) != 0) return;
    const int esz = p.resid_dtype == VTP_F32 ? 4 : 2;
#pragma unroll
    for (int it = 0; it < 8; ++it) {
        if (orow8[it] < 0 || ocol0 >= Nout) continue;
        const char* base = reinterpret_cast<const char*>(p.resid) + (orow8[it] * p.ldr + ocol0) * esz;
        asm volatile("prefetch.global.L2 [%0];" ::"l"(base));
        if (ncols * esz > 128) asm volatile("prefetch.global.L2 [%0];" ::"l"(base + 128));
    }
}

// ---- bf16 outputs: the whole 64-column unit is staged as bf16 (32 rows x 128 B, 16-byte chunks XOR-swizzled) so that
// every store instruction writes four complete 128-byte lines (64-byte partial-line writes ran ~2.5x slower).
__device__ __forceinline__ int stgb_off(int r, int chunk /*0..7, 16 B each*/) { return r * 128 + ((chunk ^ (r & 7)) << 4); }

__device__ __forceinline__ void stage_bf16(uint8_t* stg, int lane, const float (&v)[64], int c0, int nvals) {
    // packs v[0..nvals) (nvals = 32 or 64) into columns c0.. of this lane's staged row
#pragma unroll
    for (int c = 0; c < 8; ++c) {
        if (8 * c < nvals) {
            uint4 w;
            w.x = pack_bf16x2(v[8 * c], v[8 * c + 1]), w.y = pack_bf16x2(v[8 * c + 2], v[8 * c + 3]);
            w.z = pack_bf16x2(v[8 * c + 4], v[8 * c + 5]), w.w = pack_bf16x2(v[8 * c + 6], v[8 * c + 7]);
            *reinterpret_cast<uint4*>(stg + stgb_off(lane, (c0 >> 3) + c)) = w;
        }
    }
}

__device__ __forceinline__ uint32_t add_bf16x2(uint32_t a, uint32_t b) {
    return pack_bf16x2(bf16_lo(a) + bf16_lo(b), bf16_hi(a) + bf16_hi(b));
}

// cooperative store of a staged bf16 unit: dst = p.out (which=0) or p.out2 (which=1); ncols valid columns (32|64)
__device__ __forceinline__ void store_bf16(const GemmDev& p, const uint8_t* stg, int lane, const long (&orow8)[8], int ocol0,
                                           int ncols, int Nout, int which, bool has_resid) {
    const int cidx = lane & 7;
    const int c8 = 8 * cidx;
    const bool col_ok = c8 < ncols && ocol0 + c8 + 8 <= Nout;
    __nv_bfloat16* base = which ? p.out2 : reinterpret_cast<__nv_bfloat16*>(p.out);
    const long ld = which ? p.ldo2 : p.ldo;
#pragma unroll
    for (int it = 0; it < 8; ++it) {
        const int R = 4 * it + (lane >> 3);
        const long orow = orow8[it];
        if (orow < 0 || !col_ok) continue;
        uint4 w = *reinterpret_cast<const uint4*>(stg + stgb_off(R, cidx));
        if (has_resid && which == 0) {
            const uint4 rb = *reinterpret_cast<const uint4*>(reinterpret_cast<const __nv_bfloat16*>(p.resid) + orow * p.ldr + ocol0 + c8);
            w.x = add_bf16x2(w.x, rb.x), w.y = add_bf16x2(w.y, rb.y);
            w.z = add_bf16x2(w.z, rb.z), w.w = add_bf16x2(w.w, rb.w);
        }
        if (p.mask_pos && which == 0) {  // keep x where the forward activation was > 0 (bf16: sign bit clear, non-zero)
            const uint4 m = *reinterpret_cast<const uint4*>(p.mask_pos + orow * p.ldm + ocol0 + c8);
            auto keep = [](uint32_t x, uint32_t mm) {
                const uint32_t lo = ((mm & 0x7FFFu) != 0u && (mm & 0x8000u) == 0u) ? 0x0000FFFFu : 0u;
                const uint32_t hi = ((mm & 0x7FFF0000u) != 0u && (mm & 0x80000000u) == 0u) ? 0xFFFF0000u : 0u;
                return x & (lo | hi);
            };
            w.x = keep(w.x, m.x), w.y = keep(w.y, m.y), w.z = keep(w.z, m.z), w.w = keep(w.w, m.w);
        }
        *reinterpret_cast<uint4*>(base + orow * ld + ocol0 + c8) = w;
    }
}

// cooperative store of one staged 32-column half.  which = 0: main output, 1: secondary bf16 output (pre-activation)
template <bool PS>
__device__ __forceinline__ void store_half(const GemmDev& p, const float* stg, int lane, int grow0, const long (&orow8)[8],
                                           int ocol0, int h, int ncols, int Nout, int which, bool has_resid) {
    const int cidx = lane & 7;
    const int c4 = 32 * h + 4 * cidx;
    const int col = ocol0 + c4;
    const bool col_ok = c4 < ncols && col + 4 <= Nout;
#pragma unroll
    for (int it = 0; it < 8; ++it) {
        const int R = 4 * it + (lane >> 3);
        const int grow = grow0 + R;
        const long orow = orow8[it];
        if (orow < 0 || !col_ok) continue;
        float4 v = *reinterpret_cast<const float4*>(stg + stg_off(R, cidx));
        if (which == 1) {
            uint2 w;
            w.x = pack_bf16x2(v.x, v.y), w.y = pack_bf16x2(v.z, v.w);
            *reinterpret_cast<uint2*>(p.out2 + orow * p.ldo2 + col) = w;
            continue;
        }
        if constexpr (PS) {  // PixelShuffle store (decoders/pixel_decoder.py:157-160): col = c*r*r + i*r + j
            const int r = p.ps_r, gw = p.ps_gw, gh = p.ps_gh;
            const int b = grow / (gh * gw), hi = (grow / gw) % gh, wi = grow % gw;
            const int c = col / (r * r), ii = (col / r) % r, jj = col % r;
            const long idx = (((long)b * p.ps_cout + c) * (gh * r) + hi * r + ii) * (long)(gw * r) + wi * r + jj;
            if (p.out_dtype == VTP_F32) {
                *reinterpret_cast<float4*>(reinterpret_cast<float*>(p.out) + idx) = v;
            } else {
                uint2 w;
                w.x = pack_bf16x2(v.x, v.y), w.y = pack_bf16x2(v.z, v.w);
                *reinterpret_cast<uint2*>(reinterpret_cast<__nv_bfloat16*>(p.out) + idx) = w;
            }
            continue;
        }
        if (has_resid) {
            if (p.resid_dtype == VTP_F32) {
                const float4 r4 = *reinterpret_cast<const float4*>(reinterpret_cast<const float*>(p.resid) + orow * p.ldr + col);
                v.x += r4.x, v.y += r4.y, v.z += r4.z, v.w += r4.w;
            } else {
                const uint2 r2 = *reinterpret_cast<const uint2*>(reinterpret_cast<const __nv_bfloat16*>(p.resid) + orow * p.ldr + col);
                v.x += bf16_lo(r2.x), v.y += bf16_hi(r2.x), v.z += bf16_lo(r2.y), v.w += bf16_hi(r2.y);
            }
        }
        if (p.out_dtype == VTP_F32) {
            float* op = reinterpret_cast<float*>(p.out) + orow * p.ldo + col;
            if (p.accumulate) atomicAdd(reinterpret_cast<float4*>(op), v);
            else *reinterpret_cast<float4*>(op) = v;
        } else {
            uint2 w;
            w.x = pack_bf16x2(v.x, v.y), w.y = pack_bf16x2(v.z, v.w);
            *reinterpret_cast<uint2*>(reinterpret_cast<__nv_bfloat16*>(p.out) + orow * p.ldo + col) = w;
        }
    }
}

__device__ __forceinline__ void stage_half(float* stg, int lane, const float (&v)[64], int h) {
#pragma unroll
    for (int c = 0; c < 8; ++c)
        *reinterpret_cast<float4*>(stg + stg_off(lane, c)) =
            make_float4(v[32 * h + 4 * c], v[32 * h + 4 * c + 1], v[32 * h + 4 * c + 2], v[32 * h + 4 * c + 3]);
}

// one 64-column unit of a 32-row slab.  grow0 = first row of the slab, lane's own row = grow0 + lane.
// sw_half: for SwiGLU with bf16 output two adjacent packed units fill one 64-column hidden line; 0 = first, 1 = second
template <int ACT, bool PS>
__device__ __forceinline__ void epilogue_unit(const GemmDev& p, float* stg, int lane, float (&v)[64], int grow0,
                                              const long (&orow8)[8], int col0, bool has_resid, int sw_half,
                                              uint32_t (&hold)[16]) {
    const int N = p.N;
    const int grow = grow0 + lane;
    // ---- bias
    if (p.bias) {
        if (col0 + 64 <= N) {
#pragma unroll
            for (int i = 0; i < 64; i += 4) {
                float4 b = __ldg(reinterpret_cast<const float4*>(p.bias + col0 + i));
                v[i] += b.x, v[i + 1] += b.y, v[i + 2] += b.z, v[i + 3] += b.w;
            }
        } else {
#pragma unroll
            for (int i = 0; i < 64; ++i)
                if (col0 + i < N) v[i] += __ldg(p.bias + col0 + i);
        }
    }
    // the explicit rounding point is redundant when the value is only packed to bf16 afterwards (plain / ReLU store)
    const bool pack_rounds = !PS && p.out_dtype == VTP_BF16 && (ACT == VTP_ACT_NONE || ACT == VTP_ACT_RELU);
    if (p.round_bf16 && !pack_rounds) {
#pragma unroll
        for (int i = 0; i < 64; ++i) v[i] = bf16_round(v[i]);
    }
    // ---- secondary output: pre-activation, bf16
    uint8_t* stgb = reinterpret_cast<uint8_t*>(stg);
    if (p.out2) {
        stage_bf16(stgb, lane, v, 0, 64);
        __syncwarp();
        store_bf16(p, stgb, lane, orow8, col0, 64, N, 1, false);
        __syncwarp();
    }

    int ncols = 64;        // number of output columns produced by this unit
    int ocol0 = col0;      // first output column
    int Nout = N;
    // ---- activation
    if constexpr (ACT == VTP_ACT_GELU) {
#pragma unroll
        for (int i = 0; i < 64; ++i) {
            float g = gelu_erf(v[i]);
            v[i] = p.round_bf16 ? bf16_round(g) : g;
        }
    } else if constexpr (ACT == VTP_ACT_RELU) {
#pragma unroll
        for (int i = 0; i < 64; ++i) v[i] = fmaxf(v[i], 0.f);
    } else if constexpr (ACT == VTP_ACT_SWIGLU8) {
        // packed columns: [16g, 16g+8) = x1, [16g+8, 16g+16) = x2  ->  hidden[8g + i] = silu(x1) * x2
#pragma unroll
        for (int g = 0; g < 4; ++g) {
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                float x1 = v[16 * g + i], x2 = v[16 * g + 8 + i];
                float s = __fdividef(x1, 1.0f + __expf(-x1));
                if (p.round_bf16) s = bf16_round(s);
                float h = s * x2;
                v[8 * g + i] = p.round_bf16 ? bf16_round(h) : h;
            }
        }
        ncols = 32;
        ocol0 = col0 >> 1;
        Nout = N >> 1;
    } else if constexpr (ACT == VTP_ACT_ROPE) {
        const int tok = grow % p.rope_tokens;
        const int pos = tok - p.rope_prefix;
        if (col0 < p.rope_cols && pos < 0) {
            // prefix (cls) tokens are not rotated but still pass through q.to(bf16) (layers/attention.py:76-79)
#pragma unroll
            for (int i = 0; i < 64; ++i) v[i] = bf16_round(v[i]);
        }
        if (col0 < p.rope_cols && pos >= 0 && grow < p.M) {
            const uint4* sp = reinterpret_cast<const uint4*>(p.rope_sin + (long)pos * 64);
            const uint4* cp = reinterpret_cast<const uint4*>(p.rope_cos + (long)pos * 64);
            // reference: x.to(bf16); (x*cos) + (rotate_half(x)*sin), every op rounded to bf16
#pragma unroll
            for (int i = 0; i < 4; ++i) {  // columns 8i..8i+7 pair with 32+8i..
                const uint4 s_lo = __ldg(sp + i), c_lo = __ldg(cp + i), s_hi = __ldg(sp + 4 + i), c_hi = __ldg(cp + 4 + i);
                const uint32_t sl[4] = {s_lo.x, s_lo.y, s_lo.z, s_lo.w}, cl[4] = {c_lo.x, c_lo.y, c_lo.z, c_lo.w};
                const uint32_t sh[4] = {s_hi.x, s_hi.y, s_hi.z, s_hi.w}, ch[4] = {c_hi.x, c_hi.y, c_hi.z, c_hi.w};
#pragma unroll
                for (int k = 0; k < 8; ++k) {
                    const int j = 8 * i + k;
                    const float snl = (k & 1) ? bf16_hi(sl[k >> 1]) : bf16_lo(sl[k >> 1]);
                    const float csl = (k & 1) ? bf16_hi(cl[k >> 1]) : bf16_lo(cl[k >> 1]);
                    const float snh = (k & 1) ? bf16_hi(sh[k >> 1]) : bf16_lo(sh[k >> 1]);
                    const float csh = (k & 1) ? bf16_hi(ch[k >> 1]) : bf16_lo(ch[k >> 1]);
                    const float a = p.round_bf16 ? v[j] : bf16_round(v[j]);  // q.to(bf16); already rounded in bf16 mode
                    const float b = p.round_bf16 ? v[j + 32] : bf16_round(v[j + 32]);
                    v[j] = bf16_round(bf16_round(a * csl) + bf16_round((-b) * snl));
                    v[j + 32] = bf16_round(bf16_round(b * csh) + bf16_round(a * snh));
                }
            }
        }
    }
    if (!PS && p.out_dtype == VTP_BF16) {
        if constexpr (ACT == VTP_ACT_SWIGLU8) {
            // 32 hidden columns per packed unit: the pair (sw_half 0,1) forms one 64-column (128-byte) output line.
            // The first half waits in registers (the staging tile is reused by the partner's pre-activation store).
            if (sw_half == 0 && col0 + 64 < N) {
#pragma unroll
                for (int i = 0; i < 16; ++i) hold[i] = pack_bf16x2(v[2 * i], v[2 * i + 1]);
            } else {
                if (sw_half == 1) {
#pragma unroll
                    for (int c = 0; c < 4; ++c)
                        *reinterpret_cast<uint4*>(stgb + stgb_off(lane, c)) =
                            make_uint4(hold[4 * c], hold[4 * c + 1], hold[4 * c + 2], hold[4 * c + 3]);
                }
                stage_bf16(stgb, lane, v, 32 * sw_half, 32);
                __syncwarp();
                store_bf16(p, stgb, lane, orow8, ocol0 - 32 * sw_half, 32 * (sw_half + 1), Nout, 0, false);
                __syncwarp();
            }
        } else {
            stage_bf16(stgb, lane, v, 0, 64);
            __syncwarp();
            store_bf16(p, stgb, lane, orow8, ocol0, 64, Nout, 0, has_resid);
            __syncwarp();
        }
        return;
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        if (32 * h < ncols) {
            stage_half(stg, lane, v, h);
            __syncwarp();
            store_half<PS>(p, stg, lane, grow0, orow8, ocol0, h, ncols, Nout, 0, has_resid);
            __syncwarp();
        }
    }
}


// ---------------------------------------------------------------------------------------------------- fast epilogue
// The recurring shapes of the training step (qkv / proj / fc1 / fc2 forward, every dgrad) need only bias, a bf16
// rounding point, an optional residual of the output's own dtype and a store.  The generic epilogue above spends
// ~550 instructions per 64-column unit (address math, feature branches, staging read-back), misses the instruction
// cache and waits on its bias loads, which leaves short-K GEMMs epilogue-bound.  This path: lane == accumulator row; one 128-byte output row piece per lane is written into a
// 4 KB SWIZZLE_128B staging tile and leaves through ONE TMA store (clipped at the M / N tails by the tensor map);
// bias comes from a 256-byte per-warp shared tile (broadcast reads), the residual is fetched into registers one chunk
// ahead.
//   FAST: 1 bf16 out, 2 bf16 out + bf16 residual, 3 fp32 out, 4 fp32 out + fp32 residual, 5 bf16 out masked by
//   (mask_pos > 0) (ReLU backward of the LPIPS dgrads).   ACT: NONE | RELU.
// Implicit-conv GEMMs (tile = conv_TH x conv_TW pixel patch of one image) store through a 4-D NHWC tensor map: the warp's
// 32 rows are 32 / conv_TW image rows of conv_TW pixels.
//
// The fp32 accumulator tile acc_s holds BM rows of BN floats without padding; the 16-byte chunk k of row r sits at chunk
// k ^ acc_key(r), acc_key(r) = 2 (r & 3) + ((r >> 2) & 1), which only permutes the low three chunk bits.  Bank groups of
// 4 banks = 16-byte chunk index mod 8 (a row is a multiple of 128 bytes), and:
//  - epilogue reads, 16 B per lane, lane = row: a quarter-warp reads one logical chunk of rows 8a .. 8a+7, and acc_key
//    takes all 8 values on them, so the 8 reads fall into 8 distinct bank groups;
//  - the wgmma fragment dump, 8 B per lane: a half-warp writes rows 8a + 4h + (0..3) (h = half-warp), logical chunks
//    2j + ((lane >> 1) & 1) at 8-byte half (lane & 1).  The stored chunk's bits 2..1 are j ^ (r & 3) and bit 0 is
//    ((lane >> 1) & 1) ^ h, so the 8 (row, chunk) pairs of a half-warp cover the 8 bank groups once and the 16 lanes the
//    32 banks once.
// (A +4-float row padding keeps the reads conflict-free but gives the dump 2-way conflicts.)
__device__ __forceinline__ int acc_key(int r) { return ((r & 3) << 1) | ((r >> 2) & 1); }

// 32 consecutive fp32 accumulator columns [col0, col0 + 32) of the lane's row (col0 % 32 == 0; key = acc_key(row))
__device__ __forceinline__ void acc_ld32(const float* arow, int col0, int key, uint32_t (&r)[32]) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const float4 v = *reinterpret_cast<const float4*>(arow + col0 + 4 * (i ^ key));
        r[4 * i] = __float_as_uint(v.x), r[4 * i + 1] = __float_as_uint(v.y), r[4 * i + 2] = __float_as_uint(v.z),
        r[4 * i + 3] = __float_as_uint(v.w);
    }
}

// Hand-off of acc_s from the MMA warps to the epilogue warps, one mbarrier phase per tile: acc_full completes when all
// MMA warps have dumped the tile, acc_empty when all epilogue warps have read it (their stores may still be in flight).
struct AccHandoff {
    uint64_t* full;
    uint64_t* empty;
    uint32_t phase;  // parity of the current tile's phase
    __device__ __forceinline__ void wait_full() const { mbar_wait(full, phase); }
    // after this warp's last acc_s read of the tile
    __device__ __forceinline__ void release(int lane) const {
        __syncwarp();
        if (lane == 0) mbar_arrive(empty);
    }
};

// Tile index t = work_id, work_id + stride, ... decomposed as t = (ks * num_m + m) * num_n + n WITHOUT a division per tile: the
// producer is a single thread, and three runtime integer divisions per tile (~150 dependent instructions)
// would sit directly on the operand-feed path of the short-K GEMMs.
struct TileIter {
    int n, m, ks;          // current tile
    int dn, dm, dks;       // decomposition of the stride
    int nn, nm;
    __device__ __forceinline__ TileIter(int t0, int stride, int num_n, int num_m) : nn(num_n), nm(num_m) {
        n = t0 % num_n;
        const int r = t0 / num_n;
        m = r % num_m, ks = r / num_m;
        dn = stride % num_n;
        const int rs = stride / num_n;
        dm = rs % num_m, dks = rs / num_m;
    }
    __device__ __forceinline__ void next() {
        n += dn, m += dm, ks += dks;
        if (n >= nn) n -= nn, ++m;
        if (m >= nm) m -= nm, ++ks;
    }
};

// ---- SwiGLU gate in the lean epilogue (FAST 6: hidden + pre-activation outputs, FAST 7: hidden only).
// The stand-alone gate pass re-read the whole [M, 2Hs] pre-activation (539 MB per FFN forward at the bench shape, 6.6 ms of
// the step); here the epilogue warp takes the two ADJACENT 64-column packed chunks of its rows (8-interleaved w1|w2:
// columns [16g, 16g+8) = x1, [16g+8, 16g+16) = x2), stores them as the pre-activation through tmO2 and writes their 32 + 32
// hidden values  round(round(silu(x1)) * x2)  (layers/ffn.py:77-81 under autocast) into a second 32 x 128-byte staging tile
// that leaves through ONE TMA store of the [M, Hs] hidden tensor (tmO).
template <int BN, int FAST>
__device__ __forceinline__ void fast_swiglu_tile(const GemmDev& p, const CUtensorMap* tmO, const CUtensorMap* tmO2, uint8_t* stg,
                                                 uint8_t* stg2, float* bias_s, int lane, int q, const AccHandoff& ah,
                                                 const float* arow, int key, int m_blk, int n0) {
    static_assert(BN == 128, "one packed chunk pair = one 64-column hidden line per tile row");
    constexpr bool PRE = FAST == 6;
    const int m0 = m_blk * BM;
    const int N = p.N;
    ah.wait_full();
    {
#pragma unroll
        for (int j = 0; j < 2; ++j) {
            const int col0 = n0 + j * 64;
            const bool valid = col0 < N;     // warp-uniform (ragged last tile: N % 64 != 0 is clipped by the tensor maps)
            uint32_t r0[32], r1[32];
            if (valid) {
                acc_ld32(arow, j * 64, key, r0);
                acc_ld32(arow, j * 64 + 32, key, r1);
            }
            if (j == 1) ah.release(lane);
            bias_s[lane] = (p.bias && col0 + lane < N) ? __ldg(p.bias + col0 + lane) : 0.f;
            bias_s[32 + lane] = (p.bias && col0 + 32 + lane < N) ? __ldg(p.bias + col0 + 32 + lane) : 0.f;
            if (lane == 0) bulk_wait_read0();   // earlier TMA stores of this warp have finished reading both staging tiles
            __syncwarp();
            uint32_t hw[16];                    // 32 hidden values of this chunk, packed
            uint32_t xs[32];                    // the chunk's ROUNDED values regrouped: [0,16) = x1 pairs, [16,32) = x2 pairs
#pragma unroll
            for (int i = 0; i < 8; ++i) {       // 8 pieces of 8 packed columns: even pieces = x1 of a group, odd = x2
                const float4 ba = *reinterpret_cast<const float4*>(bias_s + 8 * i);
                const float4 bb = *reinterpret_cast<const float4*>(bias_s + 8 * i + 4);
                const uint32_t* r = i < 4 ? r0 + 8 * i : r1 + 8 * (i - 4);
                float v[8] = {__uint_as_float(r[0]) + ba.x, __uint_as_float(r[1]) + ba.y, __uint_as_float(r[2]) + ba.z,
                              __uint_as_float(r[3]) + ba.w, __uint_as_float(r[4]) + bb.x, __uint_as_float(r[5]) + bb.y,
                              __uint_as_float(r[6]) + bb.z, __uint_as_float(r[7]) + bb.w};
                if (!valid) {
#pragma unroll
                    for (int k = 0; k < 8; ++k) v[k] = 0.f;
                }
                uint4 w;
                w.x = pack_bf16x2(v[0], v[1]), w.y = pack_bf16x2(v[2], v[3]);
                w.z = pack_bf16x2(v[4], v[5]), w.w = pack_bf16x2(v[6], v[7]);
                if (PRE) *reinterpret_cast<uint4*>(stg + stgb_off(lane, i)) = w;
                // keep the ROUNDED values: the gate acts on the bf16 outputs of w1 / w2 (autocast)
                xs[(i & 1) * 16 + (i >> 1) * 4 + 0] = w.x, xs[(i & 1) * 16 + (i >> 1) * 4 + 1] = w.y;
                xs[(i & 1) * 16 + (i >> 1) * 4 + 2] = w.z, xs[(i & 1) * 16 + (i >> 1) * 4 + 3] = w.w;
            }
#pragma unroll
            for (int k = 0; k < 16; ++k) {
                const float a0 = bf16_lo(xs[k]), a1 = bf16_hi(xs[k]), b0 = bf16_lo(xs[16 + k]), b1 = bf16_hi(xs[16 + k]);
                const float s0 = bf16_round(__fdividef(a0, 1.0f + __expf(-a0)));
                const float s1 = bf16_round(__fdividef(a1, 1.0f + __expf(-a1)));
                hw[k] = pack_bf16x2(s0 * b0, s1 * b1);
            }
#pragma unroll
            for (int c = 0; c < 4; ++c)       // 32 hidden values = 64 bytes = chunks 4 j .. 4 j + 3 of the 128-byte hidden row
                *reinterpret_cast<uint4*>(stg2 + stgb_off(lane, 4 * j + c)) = make_uint4(hw[4 * c], hw[4 * c + 1], hw[4 * c + 2], hw[4 * c + 3]);
            if (PRE && valid) {
                fence_proxy_async_smem();
                __syncwarp();
                if (lane == 0) {
                    tma_store_2d(tmO2, stg, col0, m0 + q * 32);
                    bulk_commit();
                }
            }
        }
        fence_proxy_async_smem();
        __syncwarp();
        if (lane == 0) {
            tma_store_2d(tmO, stg2, n0 >> 1, m0 + q * 32);
            bulk_commit();
        }
    }
}

template <int BN, int ACT, int FAST>
__device__ __forceinline__ void fast_epilogue_tile(const GemmDev& p, const CUtensorMap* tmO, uint8_t* stg, float* bias_s,
                                                   int lane, int q, const AccHandoff& ah, const float* arow, int key,
                                                   int m_blk, int n0) {
    constexpr bool OF32 = FAST == 3 || FAST == 4;
    constexpr bool MASK = FAST == 5;
    constexpr bool RES = FAST == 2 || FAST == 4 || MASK;  // a second [M][N]-shaped operand read one chunk ahead
    const int m0 = m_blk * BM;
    constexpr int CW = OF32 ? 32 : 64;   // accumulator columns per 128-byte output chunk
    constexpr int TCH = BN / CW;         // chunks per tile row, all taken by this warp
    constexpr int PW = OF32 ? 4 : 8;     // columns per 16-byte piece
    const int N = p.N;
    long row = (long)m0 + q * 32 + lane;
    bool row_ok = row < p.M;
    int ctx = 0, cty = 0, cb = 0;  // conv: tile coordinates
    if (p.conv_C) {
        ctx = m_blk % p.conv_tiles_w, cty = (m_blk / p.conv_tiles_w) % p.conv_tiles_h;
        cb = m_blk / (p.conv_tiles_w * p.conv_tiles_h);
        const int r = q * 32 + lane;
        const int h = cty * p.conv_TH + r / p.conv_TW, w = ctx * p.conv_TW + r % p.conv_TW;
        row = ((long)cb * p.conv_H + h) * p.conv_W + w;
        row_ok = h < p.conv_H && cb < p.conv_B;
    }
    const char* rrow = !RES ? nullptr
                       : MASK ? reinterpret_cast<const char*>(p.mask_pos) + row * (long)p.ldm * 2
                              : reinterpret_cast<const char*>(p.resid) + row * (long)p.ldr * (OF32 ? 4 : 2);

    float b0n = 0.f, b1n = 0.f;
    uint4 rr[8];
    auto load_bias = [&](int col0) {
        if (p.bias) {
            b0n = (col0 + lane < N) ? __ldg(p.bias + col0 + lane) : 0.f;
            if (!OF32) b1n = (col0 + 32 + lane < N) ? __ldg(p.bias + col0 + 32 + lane) : 0.f;
        }
    };
    auto load_resid = [&](int col0) {
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const int col = col0 + PW * i;
            rr[i] = (row_ok && col + PW <= N) ? *reinterpret_cast<const uint4*>(rrow + (long)col * (OF32 ? 4 : 2))
                                              : make_uint4(0, 0, 0, 0);
        }
    };
    load_bias(n0);
    if (RES) {
        load_resid(n0);  // first chunk: in registers before the accumulator is waited for
#pragma unroll
        for (int j = 1; j < TCH; ++j) {  // later chunks: warm this lane's 128-byte row piece in L2
            const int col = n0 + j * CW;
            if (row_ok && col < N) asm volatile("prefetch.global.L2 [%0];" ::"l"(rrow + (long)col * (OF32 ? 4 : 2)));
        }
    }
    ah.wait_full();
#pragma unroll
    for (int c = 0; c < TCH; ++c) {
        const int col0 = n0 + c * CW;
        if (col0 >= N) break;  // warp-uniform
        const bool last = (c == TCH - 1) || (col0 + CW >= N);
        const float b0 = b0n, b1 = b1n;
        if (!last) load_bias(col0 + CW);
        uint32_t r0[32], r1[32];
        acc_ld32(arow, c * CW, key, r0);
        if (!OF32) acc_ld32(arow, c * CW + 32, key, r1);
        if (last) ah.release(lane);
        bias_s[lane] = b0;
        if (!OF32) bias_s[32 + lane] = b1;
        if (lane == 0) bulk_wait_read0();  // the previous TMA store has finished reading the staging tile
        __syncwarp();
        {
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                if constexpr (OF32) {
                    const float4 b = *reinterpret_cast<const float4*>(bias_s + 4 * i);
                    float4 v = make_float4(__uint_as_float(r0[4 * i]) + b.x, __uint_as_float(r0[4 * i + 1]) + b.y,
                                           __uint_as_float(r0[4 * i + 2]) + b.z, __uint_as_float(r0[4 * i + 3]) + b.w);
                    if (p.round_bf16) v.x = bf16_round(v.x), v.y = bf16_round(v.y), v.z = bf16_round(v.z), v.w = bf16_round(v.w);
                    if (ACT == VTP_ACT_RELU) v.x = fmaxf(v.x, 0.f), v.y = fmaxf(v.y, 0.f), v.z = fmaxf(v.z, 0.f), v.w = fmaxf(v.w, 0.f);
                    if (RES)
                        v.x += __uint_as_float(rr[i].x), v.y += __uint_as_float(rr[i].y), v.z += __uint_as_float(rr[i].z),
                            v.w += __uint_as_float(rr[i].w);
                    *reinterpret_cast<float4*>(stg + stgb_off(lane, i)) = v;
                } else {
                    const float4 ba = *reinterpret_cast<const float4*>(bias_s + 8 * i);
                    const float4 bb = *reinterpret_cast<const float4*>(bias_s + 8 * i + 4);
                    const uint32_t* r = i < 4 ? r0 + 8 * i : r1 + 8 * (i - 4);
                    float v[8] = {__uint_as_float(r[0]) + ba.x, __uint_as_float(r[1]) + ba.y, __uint_as_float(r[2]) + ba.z,
                                  __uint_as_float(r[3]) + ba.w, __uint_as_float(r[4]) + bb.x, __uint_as_float(r[5]) + bb.y,
                                  __uint_as_float(r[6]) + bb.z, __uint_as_float(r[7]) + bb.w};
                    if (ACT == VTP_ACT_RELU) {
#pragma unroll
                        for (int k = 0; k < 8; ++k) v[k] = fmaxf(v[k], 0.f);
                    }
                    uint4 w;
                    w.x = pack_bf16x2(v[0], v[1]), w.y = pack_bf16x2(v[2], v[3]);
                    w.z = pack_bf16x2(v[4], v[5]), w.w = pack_bf16x2(v[6], v[7]);
                    if (MASK) {  // keep x where the forward activation was > 0 (bf16: sign bit clear, non-zero)
                        auto keep = [](uint32_t x, uint32_t mm) {
                            const uint32_t lo = ((mm & 0x7FFFu) != 0u && (mm & 0x8000u) == 0u) ? 0x0000FFFFu : 0u;
                            const uint32_t hi = ((mm & 0x7FFF0000u) != 0u && (mm & 0x80000000u) == 0u) ? 0xFFFF0000u : 0u;
                            return x & (lo | hi);
                        };
                        w.x = keep(w.x, rr[i].x), w.y = keep(w.y, rr[i].y), w.z = keep(w.z, rr[i].z), w.w = keep(w.w, rr[i].w);
                    } else if (RES) {
                        w.x = add_bf16x2(w.x, rr[i].x), w.y = add_bf16x2(w.y, rr[i].y), w.z = add_bf16x2(w.z, rr[i].z),
                        w.w = add_bf16x2(w.w, rr[i].w);
                    }
                    *reinterpret_cast<uint4*>(stg + stgb_off(lane, i)) = w;
                }
            }
            if (RES && !last) load_resid(col0 + CW);  // in flight across the store and the next accumulator read
            fence_proxy_async_smem();
            __syncwarp();
            if (lane == 0) {
                if (p.conv_C) tma_store_4d(tmO, stg, col0, ctx * p.conv_TW, cty * p.conv_TH + q * (32 / p.conv_TW), cb);
                else tma_store_2d(tmO, stg, col0, m0 + q * 32);
                bulk_commit();
            }
        }
    }
}

// Consumer mainloop of one tile: warpgroup wg multiplies rows [64 wg, 64 wg + 64) of the tile.  One wgmma group stays in
// flight; a ring slot is released (one arrival per consumer warp) once the group that read it has completed.
template <int BN, int STAGES, int TA, int TB>
__device__ __forceinline__ void gemm_mainloop(float (&acc)[BN / 2], uint8_t* ring, uint64_t* full_bar, uint64_t* empty_bar,
                                              int& s, uint32_t& ph, int nkb, int wg, int lane) {
    constexpr int STAGE_BYTES = A_BYTES + BN * BK * 2;
    int prev = -1;
    for (int kb = 0; kb < nkb; ++kb) {
        mbar_wait(&full_bar[s], ph);
        const uint32_t a_base = smem_u32(ring + s * STAGE_BYTES) + wg * 8192;  // K- or MN-major: 64 rows of A = 8 KB
        const uint32_t b_base = smem_u32(ring + s * STAGE_BYTES + A_BYTES);
        wgmma_fence();
#pragma unroll
        for (int j = 0; j < BK / 16; ++j) {
            const uint64_t ad = TA ? wgmma_desc_sw128(a_base + j * 2048, 8192, 1024) : wgmma_desc_sw128(a_base + j * 32, 0, 1024);
            const uint64_t bd = TB ? wgmma_desc_sw128(b_base + j * 2048, 8192, 1024) : wgmma_desc_sw128(b_base + j * 32, 0, 1024);
            const uint32_t sc = (kb > 0 || j > 0) ? 1u : 0u;
            if constexpr (BN == 128) wgmma_m64n128_ss<TA, TB>(acc, ad, bd, sc);
            else wgmma_m64n64_ss<TA, TB>(acc, ad, bd, sc);
        }
        wgmma_commit();
        wgmma_wait<1>();
        fence_regs(acc);
        if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
        prev = s;
        if (++s == STAGES) s = 0, ph ^= 1;
    }
    wgmma_wait<0>();
    fence_regs(acc);
    if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
}

template <int BN, int STAGES, int ACT, bool PS, int FAST>
__global__ void __launch_bounds__(NUM_THREADS, 1)
gemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
            const __grid_constant__ CUtensorMap tmO, const __grid_constant__ CUtensorMap tmO2, const GemmDev p) {
    static_assert(BN == 64 || BN == 128, "tile width");
    constexpr int B_BYTES = BN * BK * 2;
    constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    constexpr int STG_BYTES = NUM_EPI_WARPS * STG_FLOATS * 4 * (FAST == 6 ? 2 : 1);  // FAST 6: + the hidden-tile staging
    uint8_t* ring = smem;
    float* acc_s = reinterpret_cast<float*>(ring + STAGES * STAGE_BYTES);
    float* stg_base = acc_s + BM * BN;                                                     // 4 epilogue warps x 4 KB
    float* bias_base = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(stg_base) + STG_BYTES);  // FAST only
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(bias_base) + (FAST ? NUM_EPI_WARPS * 256 : 0));
    uint64_t* empty_bar = full_bar + STAGES;
    uint64_t* acc_full = empty_bar + STAGES;
    uint64_t* acc_empty = acc_full + 1;

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int work_id = blockIdx.x;
    const int work_stride = gridDim.x;

    if (warp == 0 && lane == 0) {
        tma_prefetch_desc(&tmA);
        tma_prefetch_desc(&tmB);
        if (FAST) tma_prefetch_desc(&tmO);
        if (FAST == 6) tma_prefetch_desc(&tmO2);
        for (int s = 0; s < STAGES; ++s) mbar_init(&full_bar[s], 1), mbar_init(&empty_bar[s], NUM_MMA_WARPS);
        mbar_init(acc_full, NUM_MMA_WARPS);
        mbar_init(acc_empty, NUM_EPI_WARPS);
        fence_barrier_init();
    }
    __syncthreads();

    const int num_tiles = p.num_m_blocks * p.num_n_blocks * p.num_splits;
    // registers per thread: producer 40, MMA 144, epilogue 184 (40 + 2 * 144 + 184 = 4 * 128: the 64K register file).
    // ptxas allocates each role within its setmaxnreg count; this split compiles every instantiation without spills.
    if (warp < 4) {
        // ============================== TMA producer ==============================
        setmaxnreg_dec<40>();
        if (warp == 0 && lane == 0) {
            int s = 0;
            uint32_t ph = 0;
            TileIter ti(work_id, work_stride, p.num_n_blocks, p.num_m_blocks);
            for (int t = work_id; t < num_tiles; t += work_stride, ti.next()) {
                const int n_blk = ti.n, m_blk = ti.m, ks = ti.ks;
                const int kb0 = ks * p.kb_per_split;
                const int kb1 = min(kb0 + p.kb_per_split, p.num_k_blocks);
                const int m0 = m_blk * BM, n0 = n_blk * BN;
                // implicit conv: tile origin once per tile, (tap, channel block) advanced incrementally — the producer is ONE
                // thread and every runtime integer division in its k-loop is ~40 dependent instructions on the feed path
                int cv_x0 = 0, cv_y0 = 0, cv_b = 0, cv_c = 0, cv_dx = -1, cv_dy = -1;
                if (p.conv_C) {
                    cv_x0 = (m_blk % p.conv_tiles_w) * p.conv_TW;
                    cv_y0 = ((m_blk / p.conv_tiles_w) % p.conv_tiles_h) * p.conv_TH;
                    cv_b = m_blk / (p.conv_tiles_w * p.conv_tiles_h);
                    if (kb0 != 0) {  // (split-K never starts mid-way for conv, but stay general)
                        const int cpk = p.conv_C >> 6, tap = kb0 / cpk;
                        cv_c = (kb0 % cpk) << 6, cv_dx = tap % 3 - 1, cv_dy = tap / 3 - 1;
                    }
                }
                for (int kb = kb0; kb < kb1; ++kb) {
                    mbar_wait(&empty_bar[s], ph ^ 1);
                    uint8_t* sa = ring + s * STAGE_BYTES;
                    uint8_t* sb = sa + A_BYTES;
                    mbar_expect_tx(&full_bar[s], STAGE_BYTES);
                    const int k0 = kb * BK;
                    if (p.conv_C) {
                        tma_load_4d(sa, &tmA, &full_bar[s], cv_c, cv_x0 + cv_dx, cv_y0 + cv_dy, cv_b);
                        cv_c += 64;
                        if (cv_c == p.conv_C) {
                            cv_c = 0;
                            if (++cv_dx == 2) cv_dx = -1, ++cv_dy;
                        }
                    } else if (!p.a_mn) {
                        tma_load_2d(sa, &tmA, &full_bar[s], k0, m0);
                    } else {
                        tma_load_2d(sa, &tmA, &full_bar[s], m0, k0);
                        tma_load_2d(sa + 8192, &tmA, &full_bar[s], m0 + 64, k0);
                    }
                    if (!p.b_mn) {
                        tma_load_2d(sb, &tmB, &full_bar[s], k0, n0);
                    } else {
#pragma unroll
                        for (int i = 0; i < BN / 64; ++i) tma_load_2d(sb + i * 8192, &tmB, &full_bar[s], n0 + 64 * i, k0);
                    }
                    if (++s == STAGES) s = 0, ph ^= 1;
                }
            }
        }
    } else if (warp < 4 + NUM_MMA_WARPS) {
        // ============================== MMA consumers: wgmma mainloop, accumulator dump ==============================
        setmaxnreg_inc<144>();
        const int wg = (warp >> 2) - 1;    // consumer warpgroup: tile rows [64 wg, 64 wg + 64)
        const int tw = threadIdx.x & 127;
        int s = 0;
        uint32_t ph = 0, acc_ph = 0;
        TileIter ti(work_id, work_stride, p.num_n_blocks, p.num_m_blocks);
        for (int t = work_id; t < num_tiles; t += work_stride, ti.next()) {
            const int kb0 = ti.ks * p.kb_per_split;
            const int nkb = min(kb0 + p.kb_per_split, p.num_k_blocks) - kb0;
            float acc[BN / 2];
            if (p.a_mn) {
                if (p.b_mn) gemm_mainloop<BN, STAGES, 1, 1>(acc, ring, full_bar, empty_bar, s, ph, nkb, wg, lane);
                else gemm_mainloop<BN, STAGES, 1, 0>(acc, ring, full_bar, empty_bar, s, ph, nkb, wg, lane);
            } else {
                if (p.b_mn) gemm_mainloop<BN, STAGES, 0, 1>(acc, ring, full_bar, empty_bar, s, ph, nkb, wg, lane);
                else gemm_mainloop<BN, STAGES, 0, 0>(acc, ring, full_bar, empty_bar, s, ph, nkb, wg, lane);
            }
            // accumulators -> swizzled fp32 tile, once the epilogue warps have read the previous tile out of it
            mbar_wait(acc_empty, acc_ph ^ 1);
            {
                const int r0 = 64 * wg + 16 * (tw >> 5) + ((tw & 31) >> 2), c0 = 2 * (tw & 3);
                const int key = acc_key(r0);  // rows r0 and r0 + 8 share it
#pragma unroll
                for (int j = 0; j < BN / 8; ++j) {
                    const int off = 4 * ((2 * j + (c0 >> 2)) ^ key) + (c0 & 3);
                    *reinterpret_cast<float2*>(acc_s + r0 * BN + off) = make_float2(acc[4 * j], acc[4 * j + 1]);
                    *reinterpret_cast<float2*>(acc_s + (r0 + 8) * BN + off) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
                }
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(acc_full);
            acc_ph ^= 1;
        }
    } else {
        // ============================== epilogue warps ==============================
        setmaxnreg_inc<184>();
        const int q = warp & 3;  // row quarter of the tile: rows [32 q, 32 q + 32), lane = row
        float* stg = stg_base + q * STG_FLOATS;
        const bool has_resid = p.resid != nullptr;
        const float* arow = acc_s + (q * 32 + lane) * BN;
        const int key = acc_key(lane);
        AccHandoff ah{acc_full, acc_empty, 0};
        TileIter ti(work_id, work_stride, p.num_n_blocks, p.num_m_blocks);
        for (int t = work_id; t < num_tiles; t += work_stride, ti.next(), ah.phase ^= 1) {
            const int m_blk = ti.m, n0 = ti.n * BN;
            const int m0 = m_blk * BM;
            const int grow0 = m0 + q * 32;
            if constexpr (FAST == 6 || FAST == 7) {
                uint8_t* st1 = reinterpret_cast<uint8_t*>(stg);
                // FAST 6: second tile behind the pre-activation tiles; FAST 7: the only tile holds the hidden values
                uint8_t* st2 = FAST == 6 ? reinterpret_cast<uint8_t*>(stg_base) + (NUM_EPI_WARPS + q) * STG_FLOATS * 4 : st1;
                fast_swiglu_tile<BN, FAST>(p, &tmO, &tmO2, st1, st2, bias_base + q * 64, lane, q, ah, arow, key, m_blk, n0);
                continue;
            }
            if constexpr (FAST != 0) {
                fast_epilogue_tile<BN, ACT, FAST>(p, &tmO, reinterpret_cast<uint8_t*>(stg), bias_base + q * 64, lane, q, ah,
                                                  arow, key, m_blk, n0);
                continue;
            }
            constexpr bool sw = ACT == VTP_ACT_SWIGLU8;
            long orow8[8];  // output rows of the cooperative store pattern (row 4*it + lane/8 of this warp's slab)
#pragma unroll
            for (int it = 0; it < 8; ++it) orow8[it] = out_row(p, grow0 + 4 * it + (lane >> 3));
            // units in order: for SwiGLU the packed units (2k, 2k+1) form one full 128-byte hidden output line
            uint32_t hold[16];  // first half of a SwiGLU hidden line, kept in registers until its partner unit is done
            ah.wait_full();
#pragma unroll 1
            for (int u = 0; u < BN / 64; ++u) {
                const int col0 = n0 + u * 64;
                if (col0 >= p.N) break;  // warp-uniform
                if (has_resid)  // pull the residual lines into L2 before they are read
                    prefetch_resid_l2(p, lane, orow8, sw ? col0 >> 1 : col0, sw ? 32 : 64, sw ? p.N >> 1 : p.N);
                uint32_t r0[32], r1[32];
                acc_ld32(arow, u * 64, key, r0);
                acc_ld32(arow, u * 64 + 32, key, r1);
                if (u == BN / 64 - 1 || col0 + 64 >= p.N) ah.release(lane);
                float v[64];
#pragma unroll
                for (int i = 0; i < 32; ++i) v[i] = __uint_as_float(r0[i]), v[32 + i] = __uint_as_float(r1[i]);
                epilogue_unit<ACT, PS>(p, stg, lane, v, grow0, orow8, col0, has_resid, sw ? (u & 1) : 0, hold);
            }
        }
        if (FAST && lane == 0) bulk_wait0();  // outstanding TMA stores of this warp
    }
}

template <int BN, int STAGES, int ACT, bool PS, int FAST = 0>
static int launch_gemm(const CUtensorMap& tmA, const CUtensorMap& tmB, const GemmDev& p, cudaStream_t stream,
                       const CUtensorMap* tmO = nullptr, const CUtensorMap* tmO2 = nullptr) {
    constexpr int smem_bytes = 1024 + STAGES * (A_BYTES + BN * BK * 2) + BM * BN * 4 +
                               NUM_EPI_WARPS * STG_FLOATS * 4 * (FAST == 6 ? 2 : 1) + (FAST ? NUM_EPI_WARPS * 256 : 0) +
                               (2 * STAGES + 2) * 8;
    static_assert(smem_bytes <= 232448, "shared memory budget (227 KB per block)");
    static bool configured = false;
    if (!configured) {
        VTP_CUDA(cudaFuncSetAttribute(gemm_kernel<BN, STAGES, ACT, PS, FAST>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      smem_bytes));
        configured = true;
    }
    const int work = p.num_m_blocks * p.num_n_blocks * p.num_splits;
    const int grid = work < num_sms() ? work : num_sms();  // persistent: one CTA per SM
    gemm_kernel<BN, STAGES, ACT, PS, FAST><<<grid, NUM_THREADS, smem_bytes, stream>>>(tmA, tmB, tmO ? *tmO : tmA,
                                                                                     tmO2 ? *tmO2 : tmA, p);
    VTP_LAUNCH_CHECK();
    return VTP_OK;
}

}  // namespace vtp

using namespace vtp;

extern "C" int vtp_gemm_bf16(const vtp_gemm_args* a, vtp_stream_t stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    VTP_CHECK_ARG(a != nullptr, "gemm: null args");
    VTP_CHECK_ARG(a->M > 0 && a->N > 0 && a->K > 0, "gemm: bad shape M=%d N=%d K=%d", a->M, a->N, a->K);
    VTP_CHECK_ARG(a->A && a->B && a->out, "gemm: null pointer");
    VTP_CHECK_ARG(a->lda % 8 == 0 && a->ldb % 8 == 0, "gemm: lda/ldb must be multiples of 8 (16B TMA strides)");
    VTP_CHECK_ARG((reinterpret_cast<uintptr_t>(a->A) & 15) == 0 && (reinterpret_cast<uintptr_t>(a->B) & 15) == 0,
                  "gemm: A/B must be 16B aligned");
    VTP_CHECK_ARG((reinterpret_cast<uintptr_t>(a->out) & 15) == 0, "gemm: out must be 16B aligned");
    VTP_CHECK_ARG(a->N % 8 == 0, "gemm: N must be a multiple of 8");
    VTP_CHECK_ARG(a->out_dtype == VTP_F32 || a->out_dtype == VTP_BF16, "gemm: bad out dtype");
    VTP_CHECK_ARG(a->ldo % (a->out_dtype == VTP_F32 ? 4 : 8) == 0 || a->ps_r > 0, "gemm: ldo alignment");
    int split_k = a->split_k < 1 ? 1 : a->split_k;  // < 0: chosen below once the tile shape is known (needs accumulate)
    const bool auto_split = a->split_k < 0 && a->accumulate && a->out_dtype == VTP_F32 && a->act == VTP_ACT_NONE && !a->bias;
    VTP_CHECK_ARG(split_k == 1 || (a->accumulate && a->out_dtype == VTP_F32 && a->act == VTP_ACT_NONE && !a->bias),
                  "gemm: split_k needs accumulate=1, fp32 out, no bias/activation");
    VTP_CHECK_ARG(!a->accumulate || a->out_dtype == VTP_F32, "gemm: accumulate needs fp32 out");
    if (a->act == VTP_ACT_ROPE)
        VTP_CHECK_ARG(a->rope_sin && a->rope_cos && a->rope_tokens > 0 && a->rope_cols % 64 == 0, "gemm: bad rope args");
    if (a->act == VTP_ACT_SWIGLU8) VTP_CHECK_ARG(a->N % 16 == 0, "gemm: swiglu needs N %% 16 == 0");
    if (a->ps_r > 0)
        VTP_CHECK_ARG(a->ps_r % 4 == 0 && a->M % (a->ps_gh * a->ps_gw) == 0 && a->N == a->ps_cout * a->ps_r * a->ps_r,
                      "gemm: bad pixel-shuffle args");
    if (a->resid) VTP_CHECK_ARG(a->ldr % (a->resid_dtype == VTP_F32 ? 4 : 8) == 0, "gemm: ldr alignment");
    if (a->out2) VTP_CHECK_ARG(a->ldo2 % 8 == 0, "gemm: ldo2 alignment");

    const bool conv = a->conv_C > 0;
    if (conv) {
        VTP_CHECK_ARG(a->conv_C % 64 == 0 && a->conv_H > 0 && a->conv_W % 4 == 0 && !a->a_mn_major && a->K == 9 * a->conv_C &&
                          a->M % (a->conv_H * a->conv_W) == 0 && a->rr_group == 0 && a->ps_r == 0,
                      "gemm(conv): need C %% 64 == 0, W %% 4 == 0, K == 9*C, M == B*H*W");
    }
    if (a->mask_pos) VTP_CHECK_ARG(a->out_dtype == VTP_BF16 && a->ldm % 8 == 0, "gemm: mask_pos needs bf16 out");
    // 64-wide tiles when N fits in one (VGG conv1_x, 64-column projections), 128-wide otherwise
    int BN = a->N <= 64 ? 64 : 128;
    // lean TMA-store epilogue for the recurring shapes (see fast_epilogue_tile)
    const bool allow_fast = getenv("VTP_GEMM_NO_FAST") == nullptr;
    const bool fast_conv = conv && a->out_dtype == VTP_BF16 && !a->resid && getenv("VTP_GEMM_CONV_NO_FAST") == nullptr;
    const bool fast = allow_fast && (!conv || fast_conv) && a->rr_group == 0 && a->ps_r == 0 && !a->out2 &&
                      (!a->mask_pos || fast_conv) && !a->accumulate && split_k == 1 &&
                      (a->act == VTP_ACT_NONE || (a->act == VTP_ACT_RELU && !a->mask_pos)) &&
                      (!a->resid || a->resid_dtype == a->out_dtype);
    // SwiGLU gate in the lean epilogue (fast_swiglu_tile): bf16 hidden output [M, N/2] (+ optional bf16 pre-activation [M, N])
    const bool fast_swiglu = allow_fast && getenv("VTP_GEMM_NO_FAST_SWIGLU") == nullptr && a->act == VTP_ACT_SWIGLU8 && !conv &&
                             a->out_dtype == VTP_BF16 && a->round_bf16 && !a->resid && !a->mask_pos && !a->accumulate &&
                             split_k == 1 && a->rr_group == 0 && a->ps_r == 0 && a->ldo % 8 == 0;
    if (a->act == VTP_ACT_SWIGLU8) BN = 128;  // a warp's packed unit pair fills one 64-column hidden line
    if (auto_split) {
        // fill the persistent grid (one CTA per SM) as evenly as possible: the split with the best wave efficiency among
        // those that keep >= 8 k-blocks per work item
        const int grid = num_sms();
        const int tiles = ceil_div(a->M, BM) * ceil_div(a->N, BN);
        const int nkb = ceil_div(a->K, BK);
        double best = -1.0;
        for (int sp = 1; sp <= 64 && sp * 8 <= (nkb > 8 ? nkb : 8); ++sp) {
            const int kps = ceil_div(nkb, sp);
            const int real = ceil_div(nkb, kps);  // splits actually produced
            const long work = (long)tiles * real;
            if (sp > 1 && work > 3L * grid) break;  // more than three waves only adds pipeline fills and red.add traffic
            const double eff = (double)work / ((double)ceil_div((int)work, grid) * grid);
            if (eff > best + 0.02) best = eff, split_k = sp;
        }
    }

    GemmDev p;
    memset(&p, 0, sizeof(p));
    p.M = a->M, p.N = a->N, p.K = a->K;
    p.a_mn = a->a_mn_major ? 1 : 0, p.b_mn = a->b_mn_major ? 1 : 0;
    p.num_m_blocks = ceil_div(a->M, BM);
    p.num_n_blocks = ceil_div(a->N, BN);
    p.num_k_blocks = ceil_div(a->K, BK);
    p.kb_per_split = ceil_div(p.num_k_blocks, split_k);
    p.num_splits = ceil_div(p.num_k_blocks, p.kb_per_split);
    p.out = a->out, p.ldo = a->ldo, p.out_dtype = a->out_dtype;
    p.bias = a->bias, p.act = a->act, p.round_bf16 = a->round_bf16;
    p.resid = a->resid, p.ldr = a->ldr, p.resid_dtype = a->resid_dtype;
    p.accumulate = a->accumulate;
    p.rr_group = a->rr_group, p.rr_skip = a->rr_skip;
    p.rope_sin = reinterpret_cast<const __nv_bfloat16*>(a->rope_sin);
    p.rope_cos = reinterpret_cast<const __nv_bfloat16*>(a->rope_cos);
    p.rope_tokens = a->rope_tokens, p.rope_prefix = a->rope_prefix, p.rope_cols = a->rope_cols;
    p.ps_r = a->ps_r, p.ps_gh = a->ps_gh, p.ps_gw = a->ps_gw, p.ps_cout = a->ps_cout;
    p.out2 = reinterpret_cast<__nv_bfloat16*>(a->out2), p.ldo2 = a->ldo2;
    p.mask_pos = reinterpret_cast<const __nv_bfloat16*>(a->mask_pos), p.ldm = a->ldm;

    CUtensorMap tmA, tmB;
    if (conv) {
        const int W = a->conv_W, H = a->conv_H, Cc = a->conv_C, Bimg = a->M / (H * W);
        p.conv_C = Cc, p.conv_H = H, p.conv_W = W, p.conv_B = Bimg;
        p.conv_TW = (W % 16 == 0) ? 16 : (W % 8 == 0 ? 8 : 4);
        p.conv_TH = 128 / p.conv_TW;
        p.conv_tiles_w = W / p.conv_TW, p.conv_tiles_h = ceil_div(H, p.conv_TH);
        p.num_m_blocks = Bimg * p.conv_tiles_h * p.conv_tiles_w;
        p.M = p.num_m_blocks * 128;  // virtual rows (tile-local addressing, see out_row)
        uint64_t dims[4] = {(uint64_t)Cc, (uint64_t)W, (uint64_t)H, (uint64_t)Bimg};
        uint64_t strides[3] = {(uint64_t)Cc * 2, (uint64_t)W * Cc * 2, (uint64_t)H * W * Cc * 2};
        uint32_t box[4] = {64, (uint32_t)p.conv_TW, (uint32_t)p.conv_TH, 1};
        int rc = make_tmap_bf16(&tmA, a->A, 4, dims, strides, box);
        if (rc) return rc;
    } else {
        uint64_t dims[2], strides[1] = {(uint64_t)a->lda * 2};
        uint32_t box[2];
        if (!p.a_mn) dims[0] = a->K, dims[1] = a->M, box[0] = 64, box[1] = 128;
        else dims[0] = a->M, dims[1] = a->K, box[0] = 64, box[1] = 64;
        int rc = make_tmap_bf16(&tmA, a->A, 2, dims, strides, box);
        if (rc) return rc;
    }
    {
        uint64_t dims[2], strides[1] = {(uint64_t)a->ldb * 2};
        uint32_t box[2];
        if (!p.b_mn) dims[0] = a->K, dims[1] = a->N, box[0] = 64, box[1] = (uint32_t)BN;
        else dims[0] = a->N, dims[1] = a->K, box[0] = 64, box[1] = 64;
        int rc = make_tmap_bf16(&tmB, a->B, 2, dims, strides, box);
        if (rc) return rc;
    }
    // one instantiation per epilogue family keeps each kernel's code (and register pressure) small
    if (fast_swiglu) {
        CUtensorMap tmH, tmP;
        {
            uint64_t dims[2] = {(uint64_t)a->N / 2, (uint64_t)a->M}, strides[1] = {(uint64_t)a->ldo * 2};
            uint32_t box[2] = {64, 32};
            int rc = make_tmap(&tmH, a->out, VTP_BF16, 2, dims, strides, box);
            if (rc) return rc;
        }
        if (a->out2) {
            uint64_t dims[2] = {(uint64_t)a->N, (uint64_t)a->M}, strides[1] = {(uint64_t)a->ldo2 * 2};
            uint32_t box[2] = {64, 32};
            int rc = make_tmap(&tmP, a->out2, VTP_BF16, 2, dims, strides, box);
            if (rc) return rc;
            return launch_gemm<128, 4, VTP_ACT_SWIGLU8, false, 6>(tmA, tmB, p, stream, &tmH, &tmP);
        }
        return launch_gemm<128, 4, VTP_ACT_SWIGLU8, false, 7>(tmA, tmB, p, stream, &tmH);
    }
    if (fast) {
        CUtensorMap tmO;
        const int esz = a->out_dtype == VTP_F32 ? 4 : 2;
        int rc;
        if (conv) {  // NHWC output: the warp's 32 rows are 32 / TW image rows of TW pixels
            uint64_t dims[4] = {(uint64_t)a->N, (uint64_t)p.conv_W, (uint64_t)p.conv_H, (uint64_t)p.conv_B};
            uint64_t strides[3] = {(uint64_t)a->ldo * 2, (uint64_t)p.conv_W * a->ldo * 2, (uint64_t)p.conv_H * p.conv_W * a->ldo * 2};
            uint32_t box[4] = {64, (uint32_t)p.conv_TW, (uint32_t)(32 / p.conv_TW), 1};
            rc = make_tmap(&tmO, a->out, VTP_BF16, 4, dims, strides, box);
        } else {
            uint64_t dims[2] = {(uint64_t)a->N, (uint64_t)a->M}, strides[1] = {(uint64_t)a->ldo * esz};
            uint32_t box[2] = {(uint32_t)(128 / esz), 32};
            rc = make_tmap(&tmO, a->out, a->out_dtype, 2, dims, strides, box);
        }
        if (rc) return rc;
        const int mode = a->mask_pos ? 5 : (a->out_dtype == VTP_F32 ? 3 : 1) + (a->resid ? 1 : 0);
#define VTP_FAST_CFG(ACT_, MODE_)                                                                                     \
    return BN == 64 ? launch_gemm<64, 4, ACT_, false, MODE_>(tmA, tmB, p, stream, &tmO)                              \
                    : launch_gemm<128, 4, ACT_, false, MODE_>(tmA, tmB, p, stream, &tmO)
        if (mode == 5) VTP_FAST_CFG(VTP_ACT_NONE, 5);  // LPIPS dgrad with the ReLU mask: bf16 out, no bias / activation
#define VTP_FAST_ACT(ACT_)                                 \
    do {                                                   \
        switch (mode) {                                    \
            case 1: VTP_FAST_CFG(ACT_, 1);                 \
            case 2: VTP_FAST_CFG(ACT_, 2);                 \
            case 3: VTP_FAST_CFG(ACT_, 3);                 \
            default: VTP_FAST_CFG(ACT_, 4);                \
        }                                                  \
    } while (0)
        if (a->act == VTP_ACT_RELU) VTP_FAST_ACT(VTP_ACT_RELU);
        VTP_FAST_ACT(VTP_ACT_NONE);
#undef VTP_FAST_ACT
#undef VTP_FAST_CFG
    }
#define VTP_LAUNCH(ACT_, PS_)                                                              \
    return BN == 64 ? launch_gemm<64, 4, ACT_, PS_>(tmA, tmB, p, stream)                  \
                    : launch_gemm<128, 4, ACT_, PS_>(tmA, tmB, p, stream)
    if (a->ps_r > 0) {
        VTP_CHECK_ARG(a->act == VTP_ACT_NONE, "gemm: pixel shuffle has no activation");
        VTP_LAUNCH(VTP_ACT_NONE, true);
    }
    switch (a->act) {
        case VTP_ACT_NONE: VTP_LAUNCH(VTP_ACT_NONE, false);
        case VTP_ACT_GELU: VTP_LAUNCH(VTP_ACT_GELU, false);
        case VTP_ACT_SWIGLU8: return launch_gemm<128, 4, VTP_ACT_SWIGLU8, false>(tmA, tmB, p, stream);
        case VTP_ACT_ROPE: VTP_LAUNCH(VTP_ACT_ROPE, false);
        case VTP_ACT_RELU: VTP_LAUNCH(VTP_ACT_RELU, false);
        default: VTP_FAIL(VTP_ERR_ARG, "gemm: unknown activation %d", a->act);
    }
#undef VTP_LAUNCH
}
