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
    int B, T, H, D, prefix, HW, causal, nkt;  // nkt = number of 128-key tiles (1|2)
    int pack;  // > 0: `pack` whole sequences (T <= 64 tokens, prefix tokens included as ordinary rows) share one 128-row tile
    float scale_log2;                         // scale * log2(e)
    float scale;
};

}  // namespace vtp
