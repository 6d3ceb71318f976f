// vtp_b200 — argument block of the attention forward kernel (attention.cu).
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>

namespace vtp {

static constexpr int ATT_MAX_PREFIX = 4;

struct AttnDev {
    const __nv_bfloat16* qkv;  // [B*T][3D]
    __nv_bfloat16* out;        // [B*T][D]
    float* lse;                // [B][H][T] or null
    int B, T, H, D, prefix, HW, causal;
    int pack;  // > 0: `pack` whole sequences (T <= 64 tokens, prefix tokens included as ordinary rows) share one 128-row tile
    float scale_log2;                         // scale * log2(e)
    float scale;
};

// attention_long.cu: non-causal forward for HW = T - prefix > 256 (streaming K/V, online softmax).  `tm` is the
// tensor map of the packed qkv buffer with 64 x 128 boxes, as built by vtp_attention_fwd.
int attn_fwd_long(const CUtensorMap& tm, const AttnDev& p, cudaStream_t st);
// attention_long.cu: fp32 non-causal forward for T beyond the smem-resident attn_fwd_f32_kernel, K/V streamed in chunks
int attn_fwd_f32_tiled(const float* qkv, float* out, int B, int T, int H, cudaStream_t st);

}  // namespace vtp
