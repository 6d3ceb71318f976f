// vtp_b200 — device helpers shared by the attention backward kernels (attention_bwd.cu, attention_bwd_long.cu).
#pragma once
#include "ptx.cuh"

namespace vtp {

constexpr float LOG2E = 1.4426950408889634f;

__device__ __forceinline__ float ex2f(float x) {  // ex2.approx.ftz: no denormal slow path (exp2f() costs 4 extra instr)
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
// byte offset of bf16 element `col` (0..63) of row `row` in a 128-byte-swizzled tile of 128-byte rows (TMA SWIZZLE_128B)
__device__ __forceinline__ uint32_t sw_off(int row, int col) {
    return row * 128 + ((((col >> 3) ^ (row & 7)) << 4) | ((col & 7) << 1));
}
__device__ __forceinline__ void load_row64(const uint8_t* tile, int row, float (&f)[64]) {
#pragma unroll
    for (int c = 0; c < 8; ++c) {
        const uint4 w = *reinterpret_cast<const uint4*>(tile + sw_off(row, c * 8));
        f[c * 8 + 0] = bf16_lo(w.x), f[c * 8 + 1] = bf16_hi(w.x), f[c * 8 + 2] = bf16_lo(w.y), f[c * 8 + 3] = bf16_hi(w.y);
        f[c * 8 + 4] = bf16_lo(w.z), f[c * 8 + 5] = bf16_hi(w.z), f[c * 8 + 6] = bf16_lo(w.w), f[c * 8 + 7] = bf16_hi(w.w);
    }
}
__device__ __forceinline__ void load_grow64(const __nv_bfloat16* g, float (&f)[64]) {
    const uint4* p = reinterpret_cast<const uint4*>(g);
#pragma unroll
    for (int c = 0; c < 8; ++c) {
        const uint4 w = __ldg(p + c);
        f[c * 8 + 0] = bf16_lo(w.x), f[c * 8 + 1] = bf16_hi(w.x), f[c * 8 + 2] = bf16_lo(w.y), f[c * 8 + 3] = bf16_hi(w.y);
        f[c * 8 + 4] = bf16_lo(w.z), f[c * 8 + 5] = bf16_hi(w.z), f[c * 8 + 6] = bf16_lo(w.w), f[c * 8 + 7] = bf16_hi(w.w);
    }
}

// quad-split 64-dim dot product of row `row` of a swizzled smem tile with a bf16 row in global memory: thread c4 of the
// quad takes dims 16 c4 … 16 c4 + 15, the sum over the quad is returned to all four (every lane of the warp must call)
__device__ __forceinline__ float quad_dot(const uint8_t* tile, int row, const __nv_bfloat16* g, int c4) {
    float acc = 0.f;
#pragma unroll
    for (int c = 0; c < 2; ++c) {
        const uint4 a = *reinterpret_cast<const uint4*>(tile + sw_off(row, 16 * c4 + 8 * c));
        const uint4 w = __ldg(reinterpret_cast<const uint4*>(g + 16 * c4 + 8 * c));
        const uint32_t aw[4] = {a.x, a.y, a.z, a.w}, ww[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
        for (int e = 0; e < 4; ++e) acc += bf16_lo(aw[e]) * bf16_lo(ww[e]) + bf16_hi(aw[e]) * bf16_hi(ww[e]);
    }
    acc += __shfl_xor_sync(0xffffffffu, acc, 1);
    acc += __shfl_xor_sync(0xffffffffu, acc, 2);
    return acc;
}

// RoPEᵀ on the 16 dims of a row that a thread of the quad holds in an m64n64 accumulator fragment: g[2 jn + c] is dim
// 8 jn + 2 c4 + c, so dims d and d + 32 (jn and jn + 4) sit in the same thread
__device__ __forceinline__ void rope_bwd_frag(float (&g)[16], const __nv_bfloat16* sin_row, const __nv_bfloat16* cos_row, int c4) {
#pragma unroll
    for (int jn = 0; jn < 4; ++jn) {
        const int d = 8 * jn + 2 * c4;
        const uint32_t s_lo = __ldg(reinterpret_cast<const uint32_t*>(sin_row + d));
        const uint32_t s_hi = __ldg(reinterpret_cast<const uint32_t*>(sin_row + d + 32));
        const uint32_t c_lo = __ldg(reinterpret_cast<const uint32_t*>(cos_row + d));
        const uint32_t c_hi = __ldg(reinterpret_cast<const uint32_t*>(cos_row + d + 32));
        const float sl[2] = {bf16_lo(s_lo), bf16_hi(s_lo)}, sh[2] = {bf16_lo(s_hi), bf16_hi(s_hi)};
        const float cl[2] = {bf16_lo(c_lo), bf16_hi(c_lo)}, ch[2] = {bf16_lo(c_hi), bf16_hi(c_hi)};
#pragma unroll
        for (int c = 0; c < 2; ++c) {
            const float a = g[2 * jn + c], b = g[2 * (jn + 4) + c];
            g[2 * jn + c] = a * cl[c] + b * sh[c];
            g[2 * (jn + 4) + c] = b * ch[c] - a * sl[c];
        }
    }
}

// m64n64 accumulator fragment (element 4 jn + 2 i + c: row i of this thread, column 8 jn + 2 c4 + c) -> bf16 register A
// operands of the 4 k-steps of 16 columns (wgmma_m64n64_rs): a[kk][q] holds columns 16 kk + 8 (q >> 1) + 2 c4 + {0, 1}
// of row q & 1.  Callers select P and dS to 0 outside the valid rows and columns before packing: there lse and δ may be
// anything, so multiplying by 0 could give NaN.
__device__ __forceinline__ void pack_a(const float (&x)[32], uint32_t (&a)[4][4]) {
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
        a[kk][0] = pack_bf16x2(x[8 * kk], x[8 * kk + 1]), a[kk][1] = pack_bf16x2(x[8 * kk + 2], x[8 * kk + 3]);
        a[kk][2] = pack_bf16x2(x[8 * kk + 4], x[8 * kk + 5]), a[kk][3] = pack_bf16x2(x[8 * kk + 6], x[8 * kk + 7]);
    }
}

// Row i of an m64n64 fragment of 64-dim gradients (one token row, dims 8 jn + 2 c4 + c in this thread) to bf16 at drow:
// plus w · cls (the rank-1 term of the cls token, when cls is given), then RoPEᵀ (when sin_row is given)
__device__ __forceinline__ void store_grad_row(const float (&acc)[32], int i, float w, const __nv_bfloat16* cls,
                                               const __nv_bfloat16* sin_row, const __nv_bfloat16* cos_row,
                                               __nv_bfloat16* drow, int c4) {
    float g[16];
#pragma unroll
    for (int e = 0; e < 16; ++e) g[e] = acc[4 * (e >> 1) + 2 * i + (e & 1)];
    if (cls) {
#pragma unroll
        for (int jn = 0; jn < 8; ++jn) {
            const uint32_t x = __ldg(reinterpret_cast<const uint32_t*>(cls + 8 * jn + 2 * c4));
            g[2 * jn] += w * bf16_lo(x), g[2 * jn + 1] += w * bf16_hi(x);
        }
    }
    if (sin_row) rope_bwd_frag(g, sin_row, cos_row, c4);
#pragma unroll
    for (int jn = 0; jn < 8; ++jn)
        *reinterpret_cast<uint32_t*>(drow + 8 * jn + 2 * c4) = pack_bf16x2(g[2 * jn], g[2 * jn + 1]);
}

}  // namespace vtp
