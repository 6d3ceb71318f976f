"""Plain-torch fp64 references for the stages of the training step outside the transformer blocks, on the CPU or the
GPU (no kernels, nothing from oracle/):

gemm_ref      the lib.gemm contract for one recorded call: A / B majors and leading dimensions, bias, ACT_NONE / ACT_RELU /
              ACT_GELU (with out2), a residual, rr_group / rr_skip of either sign, pixel_shuffle, the implicit 3x3 conv
              (zero padding, NHWC, k = tap·C + c) with mask_pos, accumulate / split-K into the prefilled output, ldo wider
              than N, and the output's rounding point.  SwiGLU and RoPE epilogues belong to the blocks (block_ref) and
              are refused here.
w_fwd / w_bwd the LPIPS VGG weight layouts: k = tap·Cin + c, and the dgrad kernel (180° rotation, in / out swapped).
lpips_chain   LPIPSLoss._chunk composed from the stage references (step_ref's prep, pool, tap, pool_relu_bwd and
              img_grad kernels, gemm_ref for the 13 convs, the 12 dgrads and conv1_1's N = 32 input gradient).
ssl_lists     the teacher / student row lists and row weights of train._ssl_chunk from B, n_local and the mask list.
recon_coefs   the L1 and LPIPS coefficients of train.rec_fwd_bwd.

With fp64 inputs, lpips_chain is the exact chain rule of the LPIPS value (tests/test_stage_ref_cpu.py checks it against
fp64 autograd, and gemm_ref against F.conv2d, its input gradient, F.pixel_shuffle and explicit row maps).

tests/test_step_stages_gpu.py checks every recorded lib.gemm call per output row with block_ref.slack_k:
|got − ref| ≤ slack + k·2⁻²⁴·scale, slack = one bf16 ulp of the reference for a bf16 output (plus one of the residual
sum), scale = |A|·|B|ᵀ (+ |bias|, |residual|, |prefill|).

Bounds, against the largest value measured in one run of every case of the GPU file on an H100 80GB HBM3 (700 W
power limit):
    bound      value   measured maxima
    LIN_K      26      plain GEMM outputs: the contrastive feature gradient Gi·T_all 12.9 (fp32 out, K = B),
                       block GEMMs up to 3.6, patch embed 0.89, bottleneck 0.44, proj_in / proj_out 0.82
    WGRAD_K    72      = block_ref.WGRAD_K: split-K weight gradients accumulated into their prefilled buffers
    CONV_K     13      LPIPS forward convs 3.89 (conv10), dgrads 5.78 (conv9 dgrad, K = 9·512)
    DGRAD32_K  13      conv1_1's input gradient (N = 32, MN-major B, M = 32·256² rows)
    TAP_K      8       lpips_tap g0 4.18 on VGG activations at 256² (step_ref.LPIPS_K was set on random inputs)
    IMG_GRAD_K 4       lpips_img_grad 1.92
    CE_LOSS_K  10      the contrastive loss slot 5.0, 3.9 and 0 in three runs (fp32 atomics, B = 256 rows twice)
    lpips_loss_k       the LPIPS loss slot, bound = the number of block partials added + 64: 2 678 (33 images,
                       bound 7 904) and 5 261 (B = 256, 40 lpips_tap calls); with one atomic per warp, as lpips_tap
                       did before, the same runs gave 3 853 and 313 300 (1.9 % of Σ|terms|)
    chain_k(K) 4·⌈K/16⌉ the DINO head's dgrad and weight gradients with K ≥ 4096: head.last dgrad 671 (K = 65 536,
                       bound 16 384), head.mlp2 / head.last weight gradients 1 307 / 1 217 (K ≈ 11 136, bound 2 784)
    ACT_K      0.5     = step_ref.ACT_K: a GELU epilogue against the bf16 pre-activation it wrote to out2
"""
import math

import torch
import torch.nn.functional as F

from tests import block_ref as br
from tests import step_ref as sr

ACT_NONE, ACT_GELU, ACT_SWIGLU8, ACT_ROPE, ACT_RELU = 0, 1, 2, 3, 4   # vtp_b200.lib ACT_*

WGRAD_K, ACT_K = br.WGRAD_K, sr.ACT_K
LIN_K = 26.0
CONV_K = 13.0
DGRAD32_K = 13.0
TAP_K = 8.0          # lpips_tap g0 on VGG activations at 256² (step_ref.LPIPS_K was set on random inputs)
IMG_GRAD_K = 4.0     # lpips_img_grad at 256²
CE_LOSS_K = 10.0     # the contrastive loss slot: two softmax_ce launches of B rows each onto a prefilled scalar



def lpips_tap_atomics(P, C):
    """fp32 atomics one lpips_tap call adds into its loss slot: one per block, at most 1 024 blocks of 256 threads
    with 8 / 16 / 32 / 32 lanes per pixel at C = 64 / 128 / 256 / 512"""
    return min(-(-P * min(C // 8, 32) // 256), 1024)


def lpips_loss_k(taps):
    """Bound for the LPIPS loss slot after the lpips_tap calls `taps`: each same-signed block partial added to the
    running fp32 sum is rounded by at most half an ulp of it (≤ 2⁻²⁴·Σ|terms|), plus each lane's own fp32 sum of at
    most 64 pixels"""
    return float(sum(t["atomics"] for t in taps) + 64)


def chain_k(K):
    """Bound for a reduction whose running sums stay near Σ|terms| (same-signed operands, as the DINO head's GELU
    outputs and softmax gradients are).  The wgmma fp32 accumulator does not round to nearest: every 16-deep k-step
    truncates, losing up to an ulp of the accumulator (≤ 2 units of 2⁻²⁴·Σ|terms|) for the aligned products and as
    much for the addition, and those errors share a sign.  So k grows linearly with the chain length ⌈K/16⌉ instead of
    as its square root.  On an H100, all-positive operands give k = 40 / 215 / 1 273 / 5 965 at K = 1 024 / 4 096 /
    16 384 / 65 536 (about 1.5 per step), exactly what cuBLAS's bf16 GEMM with fp32 output gives up to K = 4 096;
    random-sign operands give 4.5 / 8.5 / 17.5 / 40."""
    return 4.0 * math.ceil(K / 16)


_CHUNK_ELEMS = 1 << 26      # fp64 elements per gathered operand block (512 MB)


# ------------------------------------------------------------------------------------------------------------- GEMM

def _mat(t, rows, cols, ld):
    """the [rows, cols] matrix with leading dimension ld starting at t's first element"""
    return torch.as_strided(t, (rows, cols), (ld, 1))


def _a_rows(call, rows):
    """A's rows `rows` as fp64 [len(rows), K] (conv: the 3x3 im2col rows, zero outside the image)"""
    A, M, K = call["A"], call["M"], call["K"]
    lda = call.get("lda") or A.stride(-2)
    if call.get("conv") is None:
        if call.get("a_mn"):
            return _mat(A, K, M, lda)[:, rows].t().double()
        return _mat(A, M, K, lda)[rows].double()
    C, H, W = call["conv"]
    assert lda == C and K == 9 * C, "conv: lda must be conv_C and K 9·conv_C"
    x = _mat(A, M, C, C)
    b, rem = rows // (H * W), rows % (H * W)
    h, w = rem // W, rem % W
    out = torch.empty(rows.numel(), K, dtype=torch.float64, device=A.device)
    for tap in range(9):
        dy, dx = divmod(tap, 3)
        hh, ww = h + dy - 1, w + dx - 1
        ok = (hh >= 0) & (hh < H) & (ww >= 0) & (ww < W)
        src = b * H * W + hh.clamp(0, H - 1) * W + ww.clamp(0, W - 1)
        out[:, tap * C:(tap + 1) * C] = x[src].double() * ok[:, None]
    return out


def _b_mat(call):
    """B as fp64 [N, K]"""
    B, N, K = call["B"], call["N"], call["K"]
    ldb = call.get("ldb") or B.stride(-2)
    return (_mat(B, K, N, ldb).t() if call.get("b_mn") else _mat(B, N, K, ldb)).double()


def out_index(call, rows):
    """flat element offsets (from out's first element) of the outputs of GEMM rows `rows`, [len(rows), N]"""
    N, out = call["N"], call["out"]
    ldo = call.get("ldo") or (out.stride(-2) if out.dim() >= 2 else N)
    cols = torch.arange(N, device=rows.device)
    ps = call.get("pixel_shuffle")
    if ps is not None:
        r, gh, gw, cout = ps
        b, rem = rows // (gh * gw), rows % (gh * gw)
        i, j = rem // gw, rem % gw
        c, sub = cols // (r * r), cols % (r * r)
        dy, dx = sub // r, sub % r
        y = i[:, None] * r + dy[None]
        return ((b[:, None] * cout + c[None]) * (gh * r) + y) * ldo + j[:, None] * r + dx[None]
    g, s = call.get("rr_group", 0), call.get("rr_skip", 0)
    orow = rows if s == 0 else (rows // g) * (g + s) + s + rows % g
    return orow[:, None] * ldo + cols[None]


def written_rows(call):
    """the GEMM rows whose output is stored (rr_skip < 0 drops the first −rr_skip rows of every group)"""
    rows = torch.arange(call["M"], device=call["out"].device)
    g, s = call.get("rr_group", 0), call.get("rr_skip", 0)
    return rows[rows % g >= -s] if s < 0 else rows


def gemm_ref(call, rows, before=None):
    """fp64 reference of the outputs of GEMM rows `rows` of one lib.gemm call (its keyword arguments plus A, B, out)
    -> dict(out=(ref, slack, scale)[, out2=(ref, slack, scale)]), each [len(rows), N]; `before`: the whole output
    tensor before the call (needed for accumulate).  Refuses the SwiGLU and RoPE epilogues (block_ref covers them)."""
    act = call.get("act", ACT_NONE)
    if act in (ACT_SWIGLU8, ACT_ROPE) or call.get("rope") is not None:
        raise NotImplementedError("gemm_ref: SwiGLU / RoPE epilogues are block_ref's")
    a, b = _a_rows(call, rows), _b_mat(call)
    y, scale = a @ b.t(), a.abs() @ b.abs().t()
    if call.get("bias") is not None:
        y, scale = y + call["bias"].double(), scale + call["bias"].double().abs()
    bf_out = call["out"].dtype == torch.bfloat16
    rnd = call.get("round_bf16", True)
    res = {}
    if call.get("out2") is not None:
        res["out2"] = (y, sr.ulp_bf16(y), scale)
    slack = sr.ulp_bf16(y) if (bf_out or rnd) else torch.zeros_like(y)
    if act == ACT_GELU:
        pre = y
        y = 0.5 * pre * (1 + torch.erf(pre / math.sqrt(2)))
        slack = 1.13 * slack + (sr.ulp_bf16(y) if (bf_out or rnd) else 0)   # |GELU'| ≤ 1.13 carries the rounding of pre
        scale = 1.13 * scale
    elif act == ACT_RELU:
        y = y.clamp(min=0)
    if call.get("resid") is not None:
        r = _mat(call["resid"], call["M"], call["N"], call.get("ldr") or call["resid"].stride(-2))[rows].double()
        y, scale = y + r, scale + r.abs()
        if bf_out:
            slack = slack + sr.ulp_bf16(y)
    if call.get("mask_pos") is not None:
        mp = call["mask_pos"]
        keep = _mat(mp, call["M"], call["N"], mp.stride(-2))[rows].double() > 0
        y, slack, scale = y * keep, slack * keep, scale * keep
    if call.get("accumulate"):
        prev = before.reshape(-1)[out_index(call, rows)].double()
        y, scale, slack = prev + y, prev.abs() + scale, torch.zeros_like(y)
    res["out"] = (y, slack, scale)
    return res


def _span(t, n):
    return torch.as_strided(t, (n,), (1,))


def gemm_check(call, rows, before=None):
    """per-row k of every output of one recorded call over GEMM rows `rows` -> {'out' | 'out2' | 'out (GELU of out2)':
    k per row}.  A GELU call with out2 is checked against GELU of its own recorded bf16 pre-activation."""
    out = call["out"]
    ks = {}
    chunk = max(1, _CHUNK_ELEMS // max(call["K"], call["N"]))
    span = _span(out, int(out_index(call, rows[-1:]).max()) + 1 if rows.numel() else 1)
    for i in range(0, rows.numel(), chunk):
        r = rows[i:i + chunk]
        ref = gemm_ref(call, r, before)
        g = span[out_index(call, r)]
        if "out2" in ref:
            ldo2 = call.get("ldo2") or call["out2"].stride(-2)
            pre = _mat(call["out2"], call["M"], call["N"], ldo2)[r]
            ks.setdefault("out2", []).append(br.slack_k(pre, *ref["out2"]))
            h = 0.5 * pre.double() * (1 + torch.erf(pre.double() / math.sqrt(2)))
            ks.setdefault("out (GELU of out2)", []).append(br.slack_k(g, h, sr.ulp_bf16(h), pre.double().abs() + 1e-30))
        else:
            ks.setdefault("out", []).append(br.slack_k(g, *ref["out"]))
    return {k: torch.cat(v) for k, v in ks.items()}


def untouched(call, before):
    """True where `out` still holds `before` outside the elements the call writes (ldo wider than N, dropped or
    skipped rows, columns outside N)"""
    out = call["out"]
    n = out.numel()
    idx = out_index(call, written_rows(call)).reshape(-1)
    mask = torch.ones(n, dtype=torch.bool, device=out.device)
    mask[idx[idx < n]] = False
    a, b = out.reshape(-1), before.reshape(-1)
    return bool(((a == b) | (a != a) & (b != b))[mask].all())


# ------------------------------------------------------------------------------------------------------------ LPIPS

VGG_CFG = [64, 64, "M", 128, 128, "M", 256, 256, 256, "M", 512, 512, 512, "M", 512, 512, 512]
TAPS = (1, 3, 6, 9, 12)


def w_fwd(w):
    """[Cout, Cin, 3, 3] -> [Cout, 9·Cin], k = tap·Cin + c (conv1_1: [64, 32], columns 27..31 zero)"""
    co, ci = w.shape[:2]
    m = w.permute(0, 2, 3, 1).reshape(co, 9 * ci)
    return F.pad(m, (0, 32 - 27)) if ci == 3 else m


def w_bwd(w):
    """the dgrad weights: conv3x3 of dY with the 180° rotated kernel, in / out channels swapped -> [Cin, 9·Cout],
    k = tap·Cout + co"""
    co, ci = w.shape[:2]
    return w.flip(2, 3).permute(1, 2, 3, 0).reshape(ci, 9 * co)


def lpips_sizes(H, W):
    sizes, h, w = [], H, W
    for c in VGG_CFG:
        if c == "M":
            h, w = h // 2, w // 2
        else:
            sizes.append((h, w))
    return sizes


def _rows(M, dev):
    return torch.arange(M, device=dev)


def vgg_features(img, vgg_w, vgg_b, rounding=True):
    """NCHW img -> (im2col [B·H·W, 32], every conv's ReLU output NHWC), each conv from the previous stage's value"""
    B, _, H, W = img.shape
    r = sr.bf16 if rounding else (lambda t: t)
    col = r(sr.lpips_prep(img))
    acts, x, h, w, ci = [], None, H, W, 0
    for c in VGG_CFG:
        if c == "M":
            x, h, w = sr.maxpool2(x), h // 2, w // 2
            continue
        M = B * h * w
        if ci == 0:
            call = dict(A=col, B=w_fwd(vgg_w[0]).to(col.dtype), out=col, M=M, N=c, K=32, act=ACT_RELU,
                        bias=vgg_b[0])
        else:
            cin = x.shape[-1]
            call = dict(A=x.reshape(M, cin), B=w_fwd(vgg_w[ci]).to(x.dtype), out=x, M=M, N=c, K=9 * cin,
                        act=ACT_RELU, bias=vgg_b[ci], conv=(cin, h, w))
        y = r(gemm_ref(call, _rows(M, img.device))["out"][0]).reshape(B, h, w, c)
        acts.append(y)
        x = y
        ci += 1
    return col, acts


def lpips_chain(rec, tgt, vgg_w, vgg_b, lin, coef, rounding=True):
    """LPIPSLoss._chunk composed from the stage references -> dict(loss, dimg, taps, dz, dcol): loss = coef Σ_images
    LPIPS, dimg its gradient w.r.t. rec (fp64 NCHW)"""
    B, _, H, W = rec.shape
    r = sr.bf16 if rounding else (lambda t: t)
    sizes = lpips_sizes(H, W)
    _, a1 = vgg_features(tgt, vgg_w, vgg_b, rounding)
    _, a0 = vgg_features(rec, vgg_w, vgg_b, rounding)
    gt, loss = {}, 0.0
    for k, ti in enumerate(TAPS):
        h, w = sizes[ti]
        C = a0[ti].shape[-1]
        t = sr.lpips_tap(a0[ti].reshape(-1, C), a1[ti].reshape(-1, C), lin[k].reshape(-1), coef / (h * w))
        gt[ti] = r(t["g0"]).reshape(B, h, w, C)
        loss = loss + t["loss"]
    n = len(vgg_w)
    dz, dzs = gt[n - 1], {}
    for i in range(n - 1, 0, -1):
        h, w = sizes[i]
        co, cin = vgg_w[i].shape[:2]
        pooled = sizes[i - 1] != (h, w)
        M = B * h * w
        call = dict(A=dz.reshape(M, co), B=w_bwd(vgg_w[i]).to(dz.dtype), out=dz, M=M, N=cin, K=9 * co,
                    conv=(co, h, w), round_bf16=False,
                    mask_pos=None if pooled else a0[i - 1].reshape(M, cin))
        dx = r(gemm_ref(call, _rows(M, rec.device))["out"][0]).reshape(B, h, w, cin)
        dz = r(sr.pool_relu_bwd(a0[i - 1], dx, gt.get(i - 1))) if pooled else dx
        dzs[i - 1] = dz
    M = B * H * W
    call = dict(A=dz.reshape(M, 64), B=w_fwd(vgg_w[0]).to(dz.dtype), out=dz, M=M, N=32, K=64, b_mn=True, ldb=32,
                round_bf16=False)
    dcol = r(gemm_ref(call, _rows(M, rec.device))["out"][0])
    return dict(loss=loss, dimg=sr.lpips_img_grad(dcol, B, H, W)[0], taps=gt, dz=dzs, dcol=dcol)


# -------------------------------------------------------------------------------------------------------------- SSL

def ssl_lists(B, n_loc, T, HW, mask_indices, masks_weight, weight, norm_B):
    """train._ssl_chunk's index lists for 2B global crops (view-major), n_loc·B local crops (crop-major) and the masked
    global patches mask_indices (flat into [2B·HW], ascending):
        teacher rows   cls of view 1 then view 0 (the reference's cat(chunk[1], chunk[0])), then the masked patch rows
        student rows   cls of every global crop in order, then the masked patch rows (row b·T + 1 + p: after the cls)
        t0 / t1        local crop (c, b) is held to both teacher cls rows of image b: t0 = b, t1 = B + b; global crop j
                       to teacher row j (= the other view's cls); masked patch i to teacher row 2B + i; t1 = −1 after
                       the local crops
        wrow           weight / (norm_B · (2 + 2·n_loc)) for every cls row, masks_weight · weight / norm_B per patch
    -> dict(teacher_rows, student_rows, t0, t1, wrow) (int64 rows, int32 t0 / t1, fp64 wrow)"""
    dev = mask_indices.device
    mi = mask_indices.long()
    B2 = 2 * B
    cls = torch.arange(B2, device=dev) * T
    m_rows = (mi // HW) * T + 1 + mi % HW
    b = torch.arange(B, device=dev)
    n_m = mi.numel()
    t0 = torch.cat([b.repeat(n_loc), torch.arange(B2, device=dev), B2 + torch.arange(n_m, device=dev)])
    t1 = torch.cat([(B + b).repeat(n_loc), torch.full((B2 + n_m,), -1, device=dev)])
    wl = weight / (norm_B * (2 + 2 * n_loc))
    wrow = torch.cat([torch.full((n_loc * B + B2,), wl, dtype=torch.float64, device=dev),
                      masks_weight.double() * (weight / norm_B)])
    return dict(teacher_rows=torch.cat([cls[B:], cls[:B], m_rows]), student_rows=torch.cat([cls, m_rows]),
                t0=t0.int(), t1=t1.int(), wrow=wrow)


# ---------------------------------------------------------------------------------------------------- reconstruction

def recon_coefs(numel, B, nB, weight, lpips_weight):
    """(L1 coefficient, LPIPS coefficient) of rec_fwd_bwd: the L1 mean over the numel/B values of each of nB images,
    and the LPIPS mean over nB images, both times the objective weight"""
    return weight / (numel // B * nB), weight * lpips_weight / nB
