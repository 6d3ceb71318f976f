"""ctypes binding of the C-ABI library (include/vtp_b200.h).  No torch types cross this boundary: only
`tensor.data_ptr()` integers, sizes and the raw CUDA stream handle.

The library is REQUIRED: there is no Python/CPU fallback for any entry point.  `load()` raises if the shared
object is missing, and every wrapper raises `VtpError` on a non-zero status.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libvtp_b200.so")

F32, BF16 = 0, 1
ACT_NONE, ACT_GELU, ACT_SWIGLU8, ACT_ROPE, ACT_RELU = 0, 1, 2, 3, 4


class VtpError(RuntimeError):
    pass


class GemmArgs(C.Structure):
    _fields_ = [
        ("M", C.c_int), ("N", C.c_int), ("K", C.c_int),
        ("A", C.c_void_p), ("lda", C.c_int), ("a_mn_major", C.c_int),
        ("B", C.c_void_p), ("ldb", C.c_int), ("b_mn_major", C.c_int),
        ("out", C.c_void_p), ("ldo", C.c_int), ("out_dtype", C.c_int),
        ("bias", C.c_void_p),
        ("act", C.c_int), ("round_bf16", C.c_int),
        ("resid", C.c_void_p), ("ldr", C.c_int), ("resid_dtype", C.c_int),
        ("accumulate", C.c_int), ("split_k", C.c_int),
        ("rr_group", C.c_int), ("rr_skip", C.c_int),
        ("rope_sin", C.c_void_p), ("rope_cos", C.c_void_p),
        ("rope_tokens", C.c_int), ("rope_prefix", C.c_int), ("rope_cols", C.c_int),
        ("ps_r", C.c_int), ("ps_gh", C.c_int), ("ps_gw", C.c_int), ("ps_cout", C.c_int),
        ("out2", C.c_void_p), ("ldo2", C.c_int),
        ("conv_C", C.c_int), ("conv_H", C.c_int), ("conv_W", C.c_int),
        ("mask_pos", C.c_void_p), ("ldm", C.c_int),
    ]


_lib = None

# name -> (restype, argtypes); every symbol declared in include/vtp_b200.h must be listed here
# (tests/test_abi.py checks the header against this table and against the built .so)
SIGNATURES: dict[str, tuple] = {
    "vtp_last_error": (C.c_char_p, []),
    "vtp_version": (C.c_int, []),
    "vtp_check_device": (C.c_int, []),
    "vtp_gemm_bf16": (C.c_int, [C.POINTER(GemmArgs), C.c_void_p]),
    "vtp_patchify": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "vtp_fill_prefix_tokens": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "vtp_apply_mask_tokens": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int,
                                        C.c_int, C.c_void_p]),
    "vtp_norm_fwd": (C.c_int, [C.c_void_p, C.c_int, C.c_long, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_float,
                               C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "vtp_split3": (C.c_int, [C.c_void_p, C.c_long, C.c_void_p, C.c_long, C.c_int, C.c_int, C.c_void_p]),
    "vtp_transpose_batched": (C.c_int, [C.c_void_p, C.c_int, C.c_long, C.c_void_p, C.c_int, C.c_long, C.c_int, C.c_int,
                                        C.c_int, C.c_void_p]),
    "vtp_gather_rows": (C.c_int, [C.c_void_p, C.c_int, C.c_long, C.c_void_p, C.c_int, C.c_long, C.c_void_p, C.c_int,
                                  C.c_int, C.c_void_p]),
    "vtp_gather_images": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_float, C.c_void_p]),
    "vtp_scatter_add_images": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_float,
                                         C.c_void_p]),
    "vtp_swiglu_fwd": (C.c_int, [C.c_void_p, C.c_void_p, C.c_long, C.c_int, C.c_void_p]),
    "vtp_rope_fwd": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_long, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "vtp_embed_tokens": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_long, C.c_int, C.c_int, C.c_void_p]),
    "vtp_l2norm_fwd": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_float,
                                 C.c_void_p]),
    "vtp_attention_fwd": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                    C.c_void_p]),
    "vtp_attention_fwd_f32": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "vtp_attention_bwd": (C.c_int, [C.c_void_p] * 7 + [C.c_int] * 5 + [C.c_void_p]),
    "vtp_attention_bwd_long": (C.c_int, [C.c_void_p] * 8 + [C.c_int] * 4 + [C.c_void_p]),
    "vtp_norm_bwd": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                               C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "vtp_swiglu_bwd": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p]),
    "vtp_gelu_bwd": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p]),
    "vtp_cast_colsum": (C.c_int, [C.c_void_p, C.c_int, C.c_long, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p]),
    "vtp_l2norm_bwd": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int,
                                 C.c_float, C.c_void_p]),
    "vtp_scatter_add_rows": (C.c_int, [C.c_void_p, C.c_int, C.c_long, C.c_void_p, C.c_long, C.c_void_p, C.c_int, C.c_int,
                                       C.c_void_p]),
    "vtp_strip_prefix": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "vtp_adamw_step": (C.c_int, [C.c_void_p] * 7 + [C.c_long] + [C.c_float] * 5 + [C.c_int, C.c_float, C.c_float,
                                                                                  C.c_void_p, C.c_void_p]),
    "vtp_hyper_tick": (C.c_int, [C.c_void_p, C.c_float, C.c_float, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]),
    "vtp_cast_f32_to_bf16": (C.c_int, [C.c_void_p, C.c_void_p, C.c_long, C.c_void_p]),
    "vtp_axpby": (C.c_int, [C.c_void_p, C.c_void_p, C.c_float, C.c_float, C.c_long, C.c_void_p]),
    "vtp_softmax_ce": (C.c_int, [C.c_void_p, C.c_long, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_long,
                                 C.c_float, C.c_void_p, C.c_void_p, C.c_void_p]),
    "vtp_dino_teacher_probs": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_float, C.c_void_p]),
    "vtp_dino_student_ce": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                                      C.c_float, C.c_void_p, C.c_void_p]),
    "vtp_weight_norm_fwd": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p]),
    "vtp_weight_norm_bwd": (C.c_int, [C.c_void_p] * 6 + [C.c_int, C.c_int, C.c_void_p]),
    "vtp_lpips_prep": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "vtp_maxpool2_fwd": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "vtp_pool_relu_bwd": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int,
                                    C.c_void_p]),
    "vtp_lpips_tap": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_long, C.c_int, C.c_float, C.c_void_p,
                                C.c_void_p]),
    "vtp_lpips_img_grad": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "vtp_recon_l1_grad": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                                    C.c_int, C.c_int, C.c_int, C.c_float, C.c_void_p]),
    "vtp_clip_gather_logits": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_long,
                                         C.c_void_p, C.c_void_p, C.c_void_p]),
    "vtp_clip_lse": (C.c_int, [C.c_void_p, C.c_void_p, C.c_long, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_float, C.c_void_p,
                               C.c_void_p, C.c_void_p, C.c_void_p]),
    "vtp_clip_grad": (C.c_int, [C.c_void_p, C.c_void_p, C.c_long, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_float,
                                C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "vtp_image_to_u8": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int,
                                  C.c_void_p]),
    "vtp_latent_stats": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "vtp_comm_alloc": (C.c_int, [C.c_long, C.POINTER(C.c_void_p)]),
    "vtp_comm_free": (C.c_int, [C.c_void_p]),
    "vtp_comm_get_handle": (C.c_int, [C.c_void_p, C.c_char_p]),
    "vtp_comm_open_handle": (C.c_int, [C.c_char_p, C.POINTER(C.c_void_p)]),
    "vtp_comm_close_handle": (C.c_int, [C.c_void_p]),
    "vtp_crop_resize_norm": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                       C.c_int, C.c_int, C.POINTER(C.c_float), C.POINTER(C.c_float), C.c_void_p]),
    "vtp_crop_augment": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                   C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.POINTER(C.c_float), C.POINTER(C.c_float),
                                   C.c_void_p]),
    "vtp_comm_barrier": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_long, C.c_void_p, C.c_void_p, C.c_void_p]),
    "vtp_probe_features": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_float, C.c_void_p,
                                     C.c_long, C.c_int, C.c_int, C.c_void_p]),
    "vtp_probe_ce": (C.c_int, [C.c_void_p, C.c_long, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                               C.c_long, C.c_void_p, C.c_void_p]),
    "vtp_probe_sgd": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_long, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int,
                                C.c_int, C.c_void_p, C.c_float, C.c_float, C.c_void_p, C.c_void_p]),
    "vtp_probe_correct": (C.c_int, [C.c_void_p, C.c_long, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                                    C.c_void_p]),
}


def load() -> C.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise VtpError(
                f"{LIB_PATH} not found — build it with `python -m vtp_b200.build` (there is no fallback path)")
        lib = C.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(lib, name)
            fn.restype = res
            fn.argtypes = args
        _lib = lib
    return _lib


LAUNCHES = 0  # number of C-ABI kernel launches issued by this process (every entry point launches exactly one kernel)


def check(status: int, what: str = "", launch: bool = True) -> None:
    global LAUNCHES
    if launch and what != "vtp_check_device":
        LAUNCHES += 1
    if status != 0:
        msg = load().vtp_last_error()
        raise VtpError(f"{what} failed with status {status}: {msg.decode() if msg else ''}")


def current_stream() -> int:
    import torch

    return torch.cuda.current_stream().cuda_stream


def _ptr(t) -> int | None:
    return None if t is None else t.data_ptr()


def _dt(t) -> int:
    import torch

    if t.dtype == torch.float32:
        return F32
    if t.dtype == torch.bfloat16:
        return BF16
    raise VtpError(f"unsupported dtype {t.dtype}")


def gemm(A, B, out, *, M: int, N: int, K: int, lda: int | None = None, ldb: int | None = None, ldo: int | None = None,
         a_mn: bool = False, b_mn: bool = False, bias=None, act: int = ACT_NONE, round_bf16: bool = True,
         resid=None, ldr: int | None = None, accumulate: bool = False, split_k: int = 1,
         rr_group: int = 0, rr_skip: int = 0, rope=None, pixel_shuffle=None, out2=None, ldo2: int | None = None,
         conv=None, mask_pos=None, stream: int | None = None) -> None:
    """out = epi(A · Bᵀ). A/B bf16 tensors (any shape; leading dims given explicitly or inferred from stride(-2))."""
    a = GemmArgs()
    a.M, a.N, a.K = M, N, K
    a.A, a.lda, a.a_mn_major = _ptr(A), (lda if lda is not None else A.stride(-2)), int(a_mn)
    a.B, a.ldb, a.b_mn_major = _ptr(B), (ldb if ldb is not None else B.stride(-2)), int(b_mn)
    a.out, a.out_dtype = _ptr(out), _dt(out)
    a.ldo = ldo if ldo is not None else (out.stride(-2) if out.dim() >= 2 else N)
    a.bias = _ptr(bias)
    a.act, a.round_bf16 = act, int(round_bf16)
    if resid is not None:
        a.resid, a.resid_dtype = _ptr(resid), _dt(resid)
        a.ldr = ldr if ldr is not None else resid.stride(-2)
    a.accumulate, a.split_k = int(accumulate), split_k
    a.rr_group, a.rr_skip = rr_group, rr_skip
    if rope is not None:
        sin, cos, tokens, prefix, cols = rope
        a.rope_sin, a.rope_cos = _ptr(sin), _ptr(cos)
        a.rope_tokens, a.rope_prefix, a.rope_cols = tokens, prefix, cols
    if pixel_shuffle is not None:
        a.ps_r, a.ps_gh, a.ps_gw, a.ps_cout = pixel_shuffle
    if out2 is not None:
        a.out2, a.ldo2 = _ptr(out2), (ldo2 if ldo2 is not None else out2.stride(-2))
    if conv is not None:
        a.conv_C, a.conv_H, a.conv_W = conv
    if mask_pos is not None:
        a.mask_pos, a.ldm = _ptr(mask_pos), mask_pos.stride(-2)
    check(load().vtp_gemm_bf16(C.byref(a), stream if stream is not None else current_stream()), "vtp_gemm_bf16")


def _st(stream):
    return stream if stream is not None else current_stream()


def patchify(img, out, p: int = 16, stream=None):
    B, Cc, H, W = img.shape
    check(load().vtp_patchify(_ptr(img), _ptr(out), _dt(out), B, Cc, H, W, p, _st(stream)), "vtp_patchify")


def fill_prefix_tokens(x, vec, B: int, tokens: int, nprefix: int, D: int, stream=None):
    check(load().vtp_fill_prefix_tokens(_ptr(x), _dt(x), _ptr(vec), B, tokens, nprefix, D, _st(stream)),
          "vtp_fill_prefix_tokens")


def apply_mask_tokens(x, mask_token, idx, HW: int, tokens: int, prefix: int, D: int, stream=None):
    check(load().vtp_apply_mask_tokens(_ptr(x), _dt(x), _ptr(mask_token), _ptr(idx), idx.numel(), HW, tokens, prefix, D,
                                       _st(stream)), "vtp_apply_mask_tokens")


OUT_F32, OUT_BF16, OUT_SPLIT3 = 0, 1, 2


def norm_fwd(x, y, w, b, eps: float, M: int, D: int, *, y_mode: int, ldx: int | None = None, rstd=None, mean=None,
             stream=None):
    check(load().vtp_norm_fwd(_ptr(x), _dt(x), ldx if ldx is not None else D, _ptr(y), y_mode, _ptr(w), _ptr(b), eps,
                              M, D, _ptr(rstd), _ptr(mean), _st(stream)), "vtp_norm_fwd")


def split3(x, out, M: int, K: int, *, b_side: bool, ldx: int | None = None, stream=None):
    check(load().vtp_split3(_ptr(x), ldx if ldx is not None else K, _ptr(out), M, K, int(b_side), _st(stream)),
          "vtp_split3")


def transpose_batched(inp, out, B: int, R: int, Cc: int, *, in_bstride: int | None = None,
                      out_bstride: int | None = None, in_offset: int = 0, stream=None):
    """in [B][R][Cc] (batch stride in_bstride elements, starting in_offset elements in) -> out [B][Cc][R]."""
    ip = inp.data_ptr() + in_offset * inp.element_size()
    check(load().vtp_transpose_batched(ip, _dt(inp), in_bstride if in_bstride is not None else R * Cc, _ptr(out),
                                       _dt(out), out_bstride if out_bstride is not None else R * Cc, B, R, Cc,
                                       _st(stream)), "vtp_transpose_batched")


def gather_rows(inp, out, idx, D: int, *, ld_in: int | None = None, ld_out: int | None = None, stream=None):
    check(load().vtp_gather_rows(_ptr(inp), _dt(inp), ld_in if ld_in is not None else D, _ptr(out), _dt(out),
                                 ld_out if ld_out is not None else D, _ptr(idx), idx.numel(), D, _st(stream)),
          "vtp_gather_rows")


def gather_images(x, out, img_idx, T: int, D: int, alpha: float = 1.0, stream=None):
    """out[i*T + t] = alpha * x[img_idx[i]*T + t]  (fp32 -> fp32; layers/block.py:207 `x[indices]`)."""
    check(load().vtp_gather_images(_ptr(x), _ptr(out), _ptr(img_idx), img_idx.numel(), T, D, alpha, _st(stream)),
          "vtp_gather_images")


def scatter_add_images(src, dst, img_idx, T: int, D: int, alpha: float = 1.0, stream=None):
    """dst[img_idx[i]*T + t] += alpha * src[i*T + t]  (fp32 dst; layers/block.py:211-217 `torch.index_add(..., alpha)`)."""
    check(load().vtp_scatter_add_images(_ptr(src), _dt(src), _ptr(dst), _ptr(img_idx), img_idx.numel(), T, D, alpha,
                                        _st(stream)), "vtp_scatter_add_images")


def _check_qkv(qkv, B: int, T: int, H: int):
    if qkv.shape[-1] != 3 * 64 * H or qkv.numel() != B * T * 3 * 64 * H:
        raise VtpError(f"attention: qkv of shape {tuple(qkv.shape)} is not [B*T={B * T}, 3*64*H={3 * 64 * H}] "
                       "(the kernels are specialised for head_dim 64)")


def attention_fwd(qkv, out, B: int, T: int, H: int, *, prefix: int, causal: bool = False, lse=None, stream=None):
    _check_qkv(qkv, B, T, H)
    check(load().vtp_attention_fwd(_ptr(qkv), _ptr(out), _ptr(lse), B, T, H, prefix, int(causal), _st(stream)),
          "vtp_attention_fwd")


def attention_fwd_f32(qkv, out, B: int, T: int, H: int, *, causal: bool = False, stream=None):
    _check_qkv(qkv, B, T, H)
    check(load().vtp_attention_fwd_f32(_ptr(qkv), _ptr(out), B, T, H, int(causal), _st(stream)),
          "vtp_attention_fwd_f32")


def embed_tokens(ids, emb, pos, out, stream=None):
    B, L = ids.shape
    check(load().vtp_embed_tokens(_ptr(ids), _ptr(emb), _ptr(pos), _ptr(out), B * L, L, emb.shape[1], _st(stream)),
          "vtp_embed_tokens")


def l2norm_fwd(x, y, M: int, D: int, eps: float = 1e-12, norm_out=None, stream=None):
    check(load().vtp_l2norm_fwd(_ptr(x), _dt(x), _ptr(y), _dt(y), _ptr(norm_out), M, D, eps, _st(stream)),
          "vtp_l2norm_fwd")


# ------------------------------------------------------------------------------------------------ training step
def attention_bwd(qkv, o, dout, lse, dqkv, B: int, T: int, H: int, *, prefix: int, causal: bool = False, rope=None,
                  stream=None):
    _check_qkv(qkv, B, T, H)
    sin, cos = (rope[0], rope[1]) if rope is not None else (None, None)
    check(load().vtp_attention_bwd(_ptr(qkv), _ptr(o), _ptr(dout), _ptr(lse), _ptr(dqkv), _ptr(sin), _ptr(cos), B, T, H,
                                   prefix, int(causal), _st(stream)), "vtp_attention_bwd")


def attention_bwd_long(qkv, o, dout, lse, delta, dqkv, B: int, T: int, H: int, *, prefix: int, rope=None, stream=None):
    """Non-causal attention backward for any length; delta: fp32 workspace [B, H, T] (overwritten)."""
    _check_qkv(qkv, B, T, H)
    sin, cos = (rope[0], rope[1]) if rope is not None else (None, None)
    check(load().vtp_attention_bwd_long(_ptr(qkv), _ptr(o), _ptr(dout), _ptr(lse), _ptr(delta), _ptr(dqkv), _ptr(sin),
                                        _ptr(cos), B, T, H, prefix, _st(stream)), "vtp_attention_bwd_long")


def norm_bwd(x, rstd, mean, w, dy, g, dw, db, M: int, D: int, gb_out=None, g_colsum=None, stream=None):
    check(load().vtp_norm_bwd(_ptr(x), _dt(x), _ptr(rstd), _ptr(mean), _ptr(w), _ptr(dy), _ptr(g), _ptr(dw), _ptr(db), M, D,
                              int(mean is not None), _ptr(gb_out), _ptr(g_colsum), _st(stream)), "vtp_norm_bwd")


def swiglu_bwd(pre, dhid, dpre, dbias, M: int, Hs: int, stream=None):
    check(load().vtp_swiglu_bwd(_ptr(pre), _ptr(dhid), _ptr(dpre), _ptr(dbias), M, Hs, _st(stream)), "vtp_swiglu_bwd")


def gelu_bwd(pre, dhid, dpre, dbias, M: int, N: int, stream=None):
    check(load().vtp_gelu_bwd(_ptr(pre), _ptr(dhid), _ptr(dpre), _ptr(dbias), M, N, _st(stream)), "vtp_gelu_bwd")


def cast_colsum(x, y, colsum, M: int, N: int, ldx: int | None = None, stream=None):
    check(load().vtp_cast_colsum(_ptr(x), _dt(x), ldx if ldx is not None else N, _ptr(y), _ptr(colsum), M, N,
                                 _st(stream)), "vtp_cast_colsum")


def l2norm_bwd(y, nrm, dy, dx, M: int, D: int, eps: float = 1e-12, stream=None):
    check(load().vtp_l2norm_bwd(_ptr(y), _dt(y), _ptr(nrm), _ptr(dy), _ptr(dx), _dt(dx), M, D, eps, _st(stream)),
          "vtp_l2norm_bwd")


def scatter_add_rows(src, dst, idx, D: int, *, ld_src: int | None = None, ld_dst: int | None = None, stream=None):
    check(load().vtp_scatter_add_rows(_ptr(src), _dt(src), ld_src if ld_src is not None else D, _ptr(dst),
                                      ld_dst if ld_dst is not None else D, _ptr(idx), idx.numel(), D, _st(stream)),
          "vtp_scatter_add_rows")


def strip_prefix(g, out, dcls, B: int, T: int, prefix: int, D: int, stream=None):
    check(load().vtp_strip_prefix(_ptr(g), _ptr(out), _ptr(dcls), B, T, prefix, D, _st(stream)), "vtp_strip_prefix")


def adamw_step(p, g, m, v, pb, teacher, teacher_b, n: int, *, lr, beta1, beta2, eps, wd, step, grad_scale=1.0,
               ema_momentum=0.0, hyper=None, stream=None):
    check(load().vtp_adamw_step(_ptr(p), _ptr(g), _ptr(m), _ptr(v), _ptr(pb), _ptr(teacher), _ptr(teacher_b), n, lr, beta1,
                                beta2, eps, wd, step, grad_scale, ema_momentum, _ptr(hyper), _st(stream)), "vtp_adamw_step")


def hyper_tick(hyper, beta1: float, beta2: float, lr_tab=None, wd_tab=None, mom_tab=None, n_tab: int = 0, stream=None):
    check(load().vtp_hyper_tick(_ptr(hyper), beta1, beta2, _ptr(lr_tab), _ptr(wd_tab), _ptr(mom_tab), n_tab, _st(stream)),
          "vtp_hyper_tick")


def cast_f32_to_bf16(x, y, n: int, stream=None):
    check(load().vtp_cast_f32_to_bf16(_ptr(x), _ptr(y), n, _st(stream)), "vtp_cast_f32_to_bf16")


def axpby(y, x, a: float, b: float, n: int, stream=None):
    check(load().vtp_axpby(_ptr(y), _ptr(x), a, b, n, _st(stream)), "vtp_axpby")


def softmax_ce(logits, R: int, Cn: int, label0: int, G, coef: float, loss_acc, dscale_acc=None, log_scale=None,
               stream=None):
    check(load().vtp_softmax_ce(_ptr(logits), logits.stride(0), R, Cn, label0, _ptr(log_scale), _ptr(G), G.stride(0), coef,
                                _ptr(loss_acc), _ptr(dscale_acc), _st(stream)), "vtp_softmax_ce")


def dino_teacher_probs(t, center, R: int, K: int, temp: float, stream=None):
    check(load().vtp_dino_teacher_probs(_ptr(t), _ptr(center), R, K, temp, _st(stream)), "vtp_dino_teacher_probs")


def dino_student_ce(s, tprobs, t0, t1, w, R: int, K: int, temp: float, loss_acc, stream=None):
    check(load().vtp_dino_student_ce(_ptr(s), _ptr(tprobs), _ptr(t0), _ptr(t1), _ptr(w), R, K, temp, _ptr(loss_acc),
                                     _st(stream)), "vtp_dino_student_ce")


def recon_l1_grad(rec, tgt, dlp, out, loss_acc, B: int, Cc: int, gh: int, gw: int, r: int, coef: float, stream=None):
    check(load().vtp_recon_l1_grad(_ptr(rec), _dt(rec), _ptr(tgt), _ptr(dlp), _ptr(out), _ptr(loss_acc), B, Cc, gh, gw, r,
                                   coef, _st(stream)), "vtp_recon_l1_grad")


def weight_norm_fwd(v, g, w, vnorm, K: int, D: int, stream=None):
    check(load().vtp_weight_norm_fwd(_ptr(v), _ptr(g), _ptr(w), _ptr(vnorm), K, D, _st(stream)), "vtp_weight_norm_fwd")


def weight_norm_bwd(v, g, vnorm, dW, dv, dg, K: int, D: int, stream=None):
    check(load().vtp_weight_norm_bwd(_ptr(v), _ptr(g), _ptr(vnorm), _ptr(dW), _ptr(dv), _ptr(dg), K, D, _st(stream)),
          "vtp_weight_norm_bwd")


# ------------------------------------------------------------------------------------------------ LPIPS
def lpips_prep(img, out, B: int, H: int, W: int, stream=None):
    check(load().vtp_lpips_prep(_ptr(img), _dt(img), _ptr(out), B, H, W, _st(stream)), "vtp_lpips_prep")


def maxpool2_fwd(x, y, B: int, H: int, W: int, Cc: int, stream=None):
    check(load().vtp_maxpool2_fwd(_ptr(x), _ptr(y), B, H, W, Cc, _st(stream)), "vtp_maxpool2_fwd")


def pool_relu_bwd(y, dpool, gtap, dz, B: int, H: int, W: int, Cc: int, stream=None):
    check(load().vtp_pool_relu_bwd(_ptr(y), _ptr(dpool), _ptr(gtap), _ptr(dz), B, H, W, Cc, _st(stream)),
          "vtp_pool_relu_bwd")


def lpips_tap(f0, f1, w, g0, P: int, Cc: int, coef: float, loss_acc, stream=None):
    check(load().vtp_lpips_tap(_ptr(f0), _ptr(f1), _ptr(w), _ptr(g0), P, Cc, coef, _ptr(loss_acc), _st(stream)),
          "vtp_lpips_tap")


def lpips_img_grad(dcol, dimg, B: int, H: int, W: int, stream=None):
    check(load().vtp_lpips_img_grad(_ptr(dcol), _ptr(dimg), B, H, W, _st(stream)), "vtp_lpips_img_grad")


def swiglu_fwd(pre, hid, M: int, Hs: int, stream=None):
    check(load().vtp_swiglu_fwd(_ptr(pre), _ptr(hid), M, Hs, _st(stream)), "vtp_swiglu_fwd")


def rope_fwd(qkv, sin, cos, rows: int, T: int, prefix: int, D: int, stream=None):
    check(load().vtp_rope_fwd(_ptr(qkv), _ptr(sin), _ptr(cos), rows, T, prefix, D, _st(stream)), "vtp_rope_fwd")


# ------------------------------------------------------------------------------------------------ contrastive exchange
def _ptr_array(ptrs):
    return (C.c_void_p * len(ptrs))(*[int(p) for p in ptrs])


def clip_gather_logits(img_ptrs, txt_ptrs, B: int, E: int, S, St, fi_all, ft_all, stream=None):
    """img_ptrs / txt_ptrs: per-rank device addresses (ints) of the L2-normalised bf16 features [B, E]."""
    world = len(img_ptrs)
    check(load().vtp_clip_gather_logits(_ptr_array(img_ptrs), _ptr_array(txt_ptrs), world, B, E, _ptr(S), _ptr(St),
                                        S.stride(0), _ptr(fi_all), _ptr(ft_all), _st(stream)), "vtp_clip_gather_logits")


def clip_lse(S, St, Bg: int, row0: int, B: int, log_scale, coef: float, lse, loss_acc, dscale_acc=None, stream=None):
    check(load().vtp_clip_lse(_ptr(S), _ptr(St), S.stride(0), Bg, row0, B, _ptr(log_scale), coef, _ptr(lse), _ptr(loss_acc),
                              _ptr(dscale_acc), _st(stream)), "vtp_clip_lse")


def clip_grad(S, St, Bg: int, row0: int, B: int, log_scale, coef: float, lse, dMi, dMt, stream=None):
    check(load().vtp_clip_grad(_ptr(S), _ptr(St), S.stride(0), Bg, dMi.stride(0), row0, B, _ptr(log_scale), coef, _ptr(lse),
                               _ptr(dMi), _ptr(dMt), _st(stream)), "vtp_clip_grad")


def comm_alloc(nbytes: int) -> int:
    p = C.c_void_p()
    check(load().vtp_comm_alloc(nbytes, C.byref(p)), "vtp_comm_alloc", launch=False)
    return int(p.value)


def comm_free(ptr: int) -> None:
    check(load().vtp_comm_free(ptr), "vtp_comm_free", launch=False)


def comm_get_handle(ptr: int) -> bytes:
    buf = C.create_string_buffer(64)
    check(load().vtp_comm_get_handle(ptr, buf), "vtp_comm_get_handle", launch=False)
    return buf.raw


def comm_open_handle(handle: bytes) -> int:
    p = C.c_void_p()
    check(load().vtp_comm_open_handle(C.create_string_buffer(handle, 64), C.byref(p)), "vtp_comm_open_handle", launch=False)
    return int(p.value)


def comm_close_handle(ptr: int) -> None:
    check(load().vtp_comm_close_handle(ptr), "vtp_comm_close_handle", launch=False)


def comm_barrier(pad_ptrs, rank: int, epoch: int, err_flag, poison=None, stream=None):
    check(load().vtp_comm_barrier(_ptr_array(pad_ptrs), len(pad_ptrs), rank, epoch, _ptr(err_flag), _ptr(poison), _st(stream)),
          "vtp_comm_barrier")


# ------------------------------------------------------------------------------------------------ linear probing
def probe_features(x, B: int, T: int, D: int, w, b, eps: float, X, *, cls_col: int, mean_col: int = -1, stream=None):
    """X[:, cls_col:+D] = final_norm(cls row of x); X[:, mean_col:+D] = mean of the normalised patch rows (mean_col >= 0).
    x fp32 [B*T, D] (the residual stream, read in place); X fp32 [B, ldX]."""
    check(load().vtp_probe_features(_ptr(x), B, T, D, _ptr(w), _ptr(b), eps, _ptr(X), X.stride(0), cls_col, mean_col,
                                    _st(stream)), "vtp_probe_features")


def probe_ce(Z, B: int, G: int, Cn: int, Cp: int, labels, loss_acc, dZ3, dbias, stream=None):
    check(load().vtp_probe_ce(_ptr(Z), Z.stride(0), B, G, Cn, Cp, _ptr(labels), _ptr(loss_acc), _ptr(dZ3), dZ3.stride(0),
                              _ptr(dbias), _st(stream)), "vtp_probe_ce")


def probe_sgd(p, g, buf, n: int, *, row_len: int, rows_per_cls: int, cls0: int, lr_table, hyper, momentum: float,
              grad_scale: float = 1.0, pb=None, stream=None):
    """lr_table fp32 [n_steps, G] (device); hyper: the step state advanced by hyper_tick."""
    check(load().vtp_probe_sgd(_ptr(p), _ptr(g), _ptr(buf), n, row_len, rows_per_cls, cls0, _ptr(lr_table),
                               lr_table.shape[1], lr_table.shape[0], _ptr(hyper), momentum, grad_scale, _ptr(pb),
                               _st(stream)), "vtp_probe_sgd")


def probe_correct(Z, B: int, G: int, Cn: int, Cp: int, labels, counts, stream=None):
    check(load().vtp_probe_correct(_ptr(Z), Z.stride(0), B, G, Cn, Cp, _ptr(labels), _ptr(counts), _st(stream)),
          "vtp_probe_correct")


# ------------------------------------------------------------------------------------------------ image / latent formats
def image_to_u8(img, sub3, div3, out, stream=None):
    """img NCHW [B,3,H,W] fp32|bf16 -> out uint8 NHWC [B,H,W,3] = clamp(((img - sub3[c]) / div3[c]) * 255, 0, 255)."""
    B, _, H, W = img.shape
    check(load().vtp_image_to_u8(_ptr(img), _dt(img), _ptr(sub3), _ptr(div3), _ptr(out), B, H, W, _st(stream)),
          "vtp_image_to_u8")


def latent_stats(lat, sum64, sumsq64, stream=None):
    B, Cc = lat.shape[0], lat.shape[1]
    HW = lat.numel() // (B * Cc)
    check(load().vtp_latent_stats(_ptr(lat), _dt(lat), B, Cc, HW, _ptr(sum64), _ptr(sumsq64), _st(stream)),
          "vtp_latent_stats")


# ------------------------------------------------------------------------------------------------ training input side
def crop_resize_norm(src_u8, src_idx, boxes, flips, out, mean=(0.485, 0.456, 0.406), std=(0.229, 0.224, 0.225), stream=None):
    """src_u8 uint8 NHWC [B,H,W,3]; src_idx int32 [N]; boxes fp32 [N,4] (x0,y0,w,h); flips uint8 [N] | None;
    out fp32 NCHW [N,3,S,S] = normalised bilinear crops."""
    B, H, W, _ = src_u8.shape
    N, _, S, _ = out.shape
    m = (C.c_float * 3)(*mean)
    sd = (C.c_float * 3)(*std)
    check(load().vtp_crop_resize_norm(_ptr(src_u8), B, H, W, _ptr(src_idx), _ptr(boxes), _ptr(flips), _ptr(out), N, S, m, sd,
                                      _st(stream)), "vtp_crop_resize_norm")


def crop_augment(src_u8, src_idx, boxes, flips, params, mean_ws, out, mean=(0.485, 0.456, 0.406), std=(0.229, 0.224, 0.225),
                 stream=None):
    """crop_resize_norm with DINOv2's photometric augmentations between the resample and the normalisation.
    params fp32 [N,8] (16-byte aligned; layout in include/vtp_b200.h), mean_ws fp32 [N] workspace; out fp32 [N,3,S,S]
    with S >= 5; the rest as in crop_resize_norm."""
    import torch

    B, H, W, _ = src_u8.shape
    N, _, S, _ = out.shape
    if src_u8.dtype != torch.uint8 or src_u8.shape[-1] != 3 or not src_u8.is_contiguous():
        raise VtpError(f"crop_augment: src must be contiguous uint8 [B,H,W,3], got {src_u8.dtype} {tuple(src_u8.shape)}")
    if out.dtype != torch.float32 or tuple(out.shape) != (N, 3, S, S) or not out.is_contiguous():
        raise VtpError(f"crop_augment: out must be contiguous fp32 [N,3,S,S], got {out.dtype} {tuple(out.shape)}")
    for name, t, dt, shape in (("src_idx", src_idx, torch.int32, (N,)), ("boxes", boxes, torch.float32, (N, 4)),
                               ("params", params, torch.float32, (N, 8)), ("mean_ws", mean_ws, torch.float32, (N,)),
                               ("flips", flips, torch.uint8, (N,))):
        if t is None and name == "flips":
            continue
        if t.dtype != dt or tuple(t.shape) != shape or not t.is_contiguous():
            raise VtpError(f"crop_augment: {name} must be contiguous {dt} {list(shape)}, got {t.dtype} {tuple(t.shape)}")
    if params.data_ptr() % 16:
        raise VtpError("crop_augment: params must be 16-byte aligned")
    m = (C.c_float * 3)(*mean)
    sd = (C.c_float * 3)(*std)
    check(load().vtp_crop_augment(_ptr(src_u8), B, H, W, _ptr(src_idx), _ptr(boxes), _ptr(flips), _ptr(params), _ptr(mean_ws),
                                  _ptr(out), N, S, m, sd, _st(stream)), "vtp_crop_augment")
