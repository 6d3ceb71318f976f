// vtp_b200 — the contrastive exchange (collective C2, SURVEY.md §8e) over NVLink peer memory, and the logit-scale
// softmax cross-entropy of OpenCLIP's ClipLoss fused behind it (vtp_hf/modeling_vtp.py:312-333 is the reference's
// logits; the loss itself is restated, SURVEY.md M3).
//
// Every rank keeps its L2-normalised image / text features [B][E] bf16 in a cudaMalloc'ed "comm" buffer whose IPC
// handle the host exchanges once (vtp_comm_*).  Per step:
//   vtp_comm_barrier          flag barrier through the peers' signal pads (release/acquire at system scope)
//   vtp_clip_gather_logits    ONE kernel: pulls the feature rows of all ranks straight out of peer memory (16-byte
//                             volatile loads over NVLink) into shared memory tiles, multiplies them on the tensor cores
//                             (warp-level mma.sync m16n8k16, fp32 accumulate) into the FULL similarity matrix
//                             S = I_all · T_allᵀ [Bg][Bg] (and Sᵀ), and leaves the gathered I_all / T_all behind as a
//                             by-product (operands of the feature-gradient GEMMs)
//   vtp_clip_lse              row log-sum-exp of exp(log_scale)·S and ·Sᵀ for ALL rows; loss and d(log_scale) of the
//                             rank's own rows
//   vtp_clip_grad             dM_i = dL/dS rows of the rank's images (row-softmax term + column-softmax term),
//                             dM_t likewise for its captions
// Because every rank holds the full Bg x Bg logits (2·Bg²·E FLOP — microseconds), the feature gradients need NO
// backward collective: dI_local = dM_i · T_all, dT_local = dM_t · I_all (two wgmma GEMMs).  The only exchange on the
// contrastive path is the forward gather, as north_star prescribes.
#include "host.h"
#include "ptx.cuh"

namespace vtp {

constexpr int CLIP_MAX_WORLD = 16;
constexpr int CT = 64;    // tile: 64 image rows x 64 text rows per CTA
constexpr int CK = 64;    // k chunk staged in shared memory
constexpr int CPAD = 72;  // shared row stride in bf16 (144 B): fragment reads hit 32 distinct banks

struct PeerTable {
    const __nv_bfloat16* img[CLIP_MAX_WORLD];
    const __nv_bfloat16* txt[CLIP_MAX_WORLD];
};

// 16-byte load that is never served from a stale L1 line (the data was written by another GPU)
__device__ __forceinline__ uint4 ld_peer16(const void* p) {
    uint4 v;
    asm volatile("ld.volatile.global.v4.u32 {%0, %1, %2, %3}, [%4];"
                 : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
                 : "l"(p)
                 : "memory");
    return v;
}

__device__ __forceinline__ void mma_bf16_16816(float (&c)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
    asm volatile(
        "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
        "{%0, %1, %2, %3};"
        : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}

// grid (ceil(Bg/64) text tiles, ceil(Bg/64) image tiles), 128 threads = 2x2 warps of 32x32
__global__ void __launch_bounds__(128) clip_gather_logits_kernel(PeerTable tbl, int B, int E, int Bg, float* __restrict__ S,
                                                                 float* __restrict__ St, long ld,
                                                                 __nv_bfloat16* __restrict__ fi_all,
                                                                 __nv_bfloat16* __restrict__ ft_all) {
    __shared__ __align__(16) __nv_bfloat16 sa[CT * CPAD];
    __shared__ __align__(16) __nv_bfloat16 sb[CT * CPAD];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int wm = warp >> 1, wn = warp & 1, g = lane >> 2, t = lane & 3;
    const int row0 = blockIdx.y * CT, col0 = blockIdx.x * CT;
    float acc[2][4][4];
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j)
#pragma unroll
            for (int k = 0; k < 4; ++k) acc[i][j][k] = 0.f;

    for (int k0 = 0; k0 < E; k0 += CK) {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int idx = tid + i * 128, r = idx >> 3, c = idx & 7;
            const int k = k0 + c * 8;
            uint4 va = make_uint4(0, 0, 0, 0), vb = make_uint4(0, 0, 0, 0);
            const int gr = row0 + r, gc = col0 + r;
            if (gr < Bg && k < E) {
                const int rk = gr / B, lr = gr - rk * B;
                va = ld_peer16(tbl.img[rk] + (long)lr * E + k);
                if (blockIdx.x == 0) *reinterpret_cast<uint4*>(fi_all + (long)gr * E + k) = va;
            }
            if (gc < Bg && k < E) {
                const int rk = gc / B, lr = gc - rk * B;
                vb = ld_peer16(tbl.txt[rk] + (long)lr * E + k);
                if (blockIdx.y == 0) *reinterpret_cast<uint4*>(ft_all + (long)gc * E + k) = vb;
            }
            *reinterpret_cast<uint4*>(sa + r * CPAD + c * 8) = va;
            *reinterpret_cast<uint4*>(sb + r * CPAD + c * 8) = vb;
        }
        __syncthreads();
#pragma unroll
        for (int kk = 0; kk < CK; kk += 16) {
            uint32_t af[2][4], bfr[4][2];
#pragma unroll
            for (int mt = 0; mt < 2; ++mt) {
                const __nv_bfloat16* p = sa + (wm * 32 + mt * 16 + g) * CPAD + kk + 2 * t;
                af[mt][0] = *reinterpret_cast<const uint32_t*>(p);
                af[mt][1] = *reinterpret_cast<const uint32_t*>(p + 8 * CPAD);
                af[mt][2] = *reinterpret_cast<const uint32_t*>(p + 8);
                af[mt][3] = *reinterpret_cast<const uint32_t*>(p + 8 * CPAD + 8);
            }
#pragma unroll
            for (int nt = 0; nt < 4; ++nt) {
                const __nv_bfloat16* p = sb + (wn * 32 + nt * 8 + g) * CPAD + kk + 2 * t;
                bfr[nt][0] = *reinterpret_cast<const uint32_t*>(p);
                bfr[nt][1] = *reinterpret_cast<const uint32_t*>(p + 8);
            }
#pragma unroll
            for (int mt = 0; mt < 2; ++mt)
#pragma unroll
                for (int nt = 0; nt < 4; ++nt) mma_bf16_16816(acc[mt][nt], af[mt], bfr[nt]);
        }
        __syncthreads();
    }
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int nt = 0; nt < 4; ++nt)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int r = row0 + wm * 32 + mt * 16 + g + 8 * h;
                const int c = col0 + wn * 32 + nt * 8 + 2 * t;
#pragma unroll
                for (int e = 0; e < 2; ++e)
                    if (r < Bg && c + e < Bg) {
                        const float v = acc[mt][nt][2 * h + e];
                        S[(long)r * ld + c + e] = v;
                        St[(long)(c + e) * ld + r] = v;
                    }
            }
}

__device__ __forceinline__ float blk_reduce(float v, float* sh, bool is_max) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
    v = is_max ? warp_max(v) : warp_sum(v);
    __syncthreads();
    if (lane == 0) sh[warp] = v;
    __syncthreads();
    float r = (threadIdx.x < nw) ? sh[threadIdx.x] : (is_max ? -INFINITY : 0.f);
    if (warp == 0) {
        r = is_max ? warp_max(r) : warp_sum(r);
        if (lane == 0) sh[0] = r;
    }
    __syncthreads();
    return sh[0];
}

// grid 2*Bg: block (d, r) reduces row r of S (d = 0: image -> text) or of Sᵀ (d = 1); lse[d*Bg + r].  Rows of this
// rank ([row0, row0+B)) also add their loss term and d(log_scale) term.
__global__ void __launch_bounds__(256) clip_lse_kernel(const float* __restrict__ S, const float* __restrict__ St, long ld,
                                                       int Bg, int row0, int B, const float* __restrict__ log_scale,
                                                       float coef, float* __restrict__ lse, float* __restrict__ loss_acc,
                                                       float* __restrict__ dscale_acc) {
    __shared__ float sh[32];
    const int d = blockIdx.x / Bg, r = blockIdx.x - d * Bg;
    const float* row = (d ? St : S) + (long)r * ld;
    const float sc = __expf(*log_scale);
    float m = -INFINITY;
    for (int c = threadIdx.x; c < Bg; c += blockDim.x) m = fmaxf(m, sc * row[c]);
    m = blk_reduce(m, sh, true);
    float s = 0.f;
    for (int c = threadIdx.x; c < Bg; c += blockDim.x) s += __expf(sc * row[c] - m);
    s = blk_reduce(s, sh, false);
    const float l = m + logf(s);
    if (threadIdx.x == 0) lse[blockIdx.x] = l;
    if (r < row0 || r >= row0 + B) return;
    float ds = 0.f;
    for (int c = threadIdx.x; c < Bg; c += blockDim.x) {
        const float x = sc * row[c];
        ds += coef * (__expf(x - l) - (c == r ? 1.f : 0.f)) * x;
    }
    ds = blk_reduce(ds, sh, false);
    if (threadIdx.x == 0) {
        atomicAdd(loss_acc, coef * (l - sc * row[r]));
        if (dscale_acc) atomicAdd(dscale_acc, ds);
    }
}

// grid 2*B: block (d, b): global row rg = row0 + b of S (d = 0) / Sᵀ (d = 1).
//   dM[d][b][c] = coef·e^s·( softmax_row(rg)[c] + softmax_col(c)[rg] − 2·δ(c == rg) ),  zero for c in [Bg, Bgp)
// i.e. d( Σ_ranks L_local ) / dS restricted to the rank's own rows: its row-direction CE plus the column-direction CE
// of every caption (image) against this image (caption).
__global__ void __launch_bounds__(256) clip_grad_kernel(const float* __restrict__ S, const float* __restrict__ St, long ld,
                                                        int Bg, int Bgp, int row0, int B,
                                                        const float* __restrict__ log_scale, float coef,
                                                        const float* __restrict__ lse, __nv_bfloat16* __restrict__ dMi,
                                                        __nv_bfloat16* __restrict__ dMt) {
    const int d = blockIdx.x / B, b = blockIdx.x - d * B, rg = row0 + b;
    const float* row = (d ? St : S) + (long)rg * ld;
    const float* lse_own = lse + (long)d * Bg;
    const float* lse_oth = lse + (long)(1 - d) * Bg;
    __nv_bfloat16* out = (d ? dMt : dMi) + (long)b * Bgp;
    const float sc = __expf(*log_scale), l = lse_own[rg], k = coef * sc;
    for (int c = threadIdx.x; c < Bgp; c += blockDim.x) {
        float v = 0.f;
        if (c < Bg) {
            const float x = sc * row[c];
            v = k * (__expf(x - l) + __expf(x - lse_oth[c]) - (c == rg ? 2.f : 0.f));
        }
        out[c] = __float2bfloat16_rn(v);
    }
}

// ------------------------------------------------------------------------------------------------ flag barrier
// pads[p] = signal pad of rank p (uint64 [world]); thread p tells rank p "rank `rank` reached `epoch`" and waits
// until rank p has told us the same.  Bounded wait: after ~20 s *err = 1 instead of hanging the GPU, and *poison (the
// caller's loss slot, read back with the step's result) becomes NaN so that the time-out reaches the host on the hot
// path without an extra synchronisation: whatever consumed stale peer features afterwards is flagged with it.
__global__ void comm_barrier_kernel(PeerTable pads, int world, int rank, unsigned long long epoch, int* __restrict__ err,
                                    float* __restrict__ poison) {
    const int p = threadIdx.x;
    if (p >= world) return;
    __threadfence_system();
    unsigned long long* theirs = reinterpret_cast<unsigned long long*>(const_cast<__nv_bfloat16*>(pads.img[p])) + rank;
    asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(theirs), "l"(epoch) : "memory");
    const unsigned long long* mine = reinterpret_cast<const unsigned long long*>(pads.img[rank]) + p;
    unsigned long long t0, t1, v;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
    for (;;) {
        asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(mine) : "memory");
        if (v >= epoch) break;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1));
        if (t1 - t0 > 20000000000ull) {
            *err = 1;
            if (poison) *poison = __int_as_float(0x7fc00000);
            break;
        }
        __nanosleep(200);
    }
}

}  // namespace vtp

using namespace vtp;

static int fill_table(PeerTable& tbl, const void* const* a, const void* const* b, int world) {
    for (int i = 0; i < CLIP_MAX_WORLD; ++i) tbl.img[i] = tbl.txt[i] = nullptr;
    for (int i = 0; i < world; ++i) {
        if (!a[i] || (b && !b[i])) return -1;
        tbl.img[i] = (const __nv_bfloat16*)a[i];
        tbl.txt[i] = b ? (const __nv_bfloat16*)b[i] : nullptr;
    }
    return 0;
}

extern "C" int vtp_clip_gather_logits(const void* const* img_ptrs, const void* const* txt_ptrs, int world, int B, int E,
                                      float* S, float* St, long ld, void* fi_all, void* ft_all, vtp_stream_t st) {
    VTP_CHECK_ARG(img_ptrs && txt_ptrs && S && St && fi_all && ft_all, "clip_gather_logits: null pointer");
    VTP_CHECK_ARG(world >= 1 && world <= CLIP_MAX_WORLD && B > 0 && E > 0 && E % 8 == 0 && ld >= (long)world * B,
                  "clip_gather_logits: bad sizes (world<=%d, E %% 8 == 0, ld >= world*B)", CLIP_MAX_WORLD);
    PeerTable tbl;
    VTP_CHECK_ARG(fill_table(tbl, img_ptrs, txt_ptrs, world) == 0, "clip_gather_logits: null peer pointer");
    const int Bg = world * B, tiles = ceil_div(Bg, CT);
    clip_gather_logits_kernel<<<dim3(tiles, tiles), 128, 0, (cudaStream_t)st>>>(tbl, B, E, Bg, S, St, ld,
                                                                               (__nv_bfloat16*)fi_all, (__nv_bfloat16*)ft_all);
    VTP_LAUNCH_CHECK();
    return VTP_OK;
}

extern "C" int vtp_clip_lse(const float* S, const float* St, long ld, int Bg, int row0, int B, const float* log_scale,
                            float coef, float* lse, float* loss_acc, float* dscale_acc, vtp_stream_t st) {
    VTP_CHECK_ARG(S && St && log_scale && lse && loss_acc && Bg > 0 && B > 0 && row0 >= 0 && row0 + B <= Bg && ld >= Bg,
                  "clip_lse: bad args");
    clip_lse_kernel<<<2 * Bg, 256, 0, (cudaStream_t)st>>>(S, St, ld, Bg, row0, B, log_scale, coef, lse, loss_acc, dscale_acc);
    VTP_LAUNCH_CHECK();
    return VTP_OK;
}

extern "C" int vtp_clip_grad(const float* S, const float* St, long ld, int Bg, int Bgp, int row0, int B,
                             const float* log_scale, float coef, const float* lse, void* dMi, void* dMt, vtp_stream_t st) {
    VTP_CHECK_ARG(S && St && log_scale && lse && dMi && dMt && Bg > 0 && Bgp >= Bg && B > 0 && row0 >= 0 && row0 + B <= Bg &&
                      ld >= Bg,
                  "clip_grad: bad args");
    clip_grad_kernel<<<2 * B, 256, 0, (cudaStream_t)st>>>(S, St, ld, Bg, Bgp, row0, B, log_scale, coef, lse,
                                                         (__nv_bfloat16*)dMi, (__nv_bfloat16*)dMt);
    VTP_LAUNCH_CHECK();
    return VTP_OK;
}

// ------------------------------------------------------------------------------------------------ peer-memory plumbing
extern "C" int vtp_comm_alloc(long bytes, void** ptr) {
    VTP_CHECK_ARG(ptr && bytes > 0, "comm_alloc: bad args");
    VTP_CUDA(cudaMalloc(ptr, (size_t)bytes));
    VTP_CUDA(cudaMemset(*ptr, 0, (size_t)bytes));
    VTP_CUDA(cudaDeviceSynchronize());
    return VTP_OK;
}
extern "C" int vtp_comm_free(void* ptr) {
    if (ptr) VTP_CUDA(cudaFree(ptr));
    return VTP_OK;
}
extern "C" int vtp_comm_get_handle(void* ptr, unsigned char* handle64) {
    VTP_CHECK_ARG(ptr && handle64, "comm_get_handle: bad args");
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
    cudaIpcMemHandle_t h;
    VTP_CUDA(cudaIpcGetMemHandle(&h, ptr));
    memcpy(handle64, &h, 64);
    return VTP_OK;
}
extern "C" int vtp_comm_open_handle(const unsigned char* handle64, void** peer_ptr) {
    VTP_CHECK_ARG(handle64 && peer_ptr, "comm_open_handle: bad args");
    cudaIpcMemHandle_t h;
    memcpy(&h, handle64, 64);
    VTP_CUDA(cudaIpcOpenMemHandle(peer_ptr, h, cudaIpcMemLazyEnablePeerAccess));
    return VTP_OK;
}
extern "C" int vtp_comm_close_handle(void* peer_ptr) {
    if (peer_ptr) VTP_CUDA(cudaIpcCloseMemHandle(peer_ptr));
    return VTP_OK;
}
extern "C" int vtp_comm_barrier(const void* const* pad_ptrs, int world, int rank, long epoch, int* err_flag,
                                float* poison, vtp_stream_t st) {
    VTP_CHECK_ARG(pad_ptrs && err_flag && world >= 1 && world <= CLIP_MAX_WORLD && rank >= 0 && rank < world && epoch > 0,
                  "comm_barrier: bad args");
    PeerTable tbl;
    VTP_CHECK_ARG(fill_table(tbl, pad_ptrs, nullptr, world) == 0, "comm_barrier: null pad pointer");
    comm_barrier_kernel<<<1, 32, 0, (cudaStream_t)st>>>(tbl, world, rank, (unsigned long long)epoch, err_flag, poison);
    VTP_LAUNCH_CHECK();
    return VTP_OK;
}
