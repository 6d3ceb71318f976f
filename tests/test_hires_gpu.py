"""Images above 256x256 (more than 256 patch tokens): the streaming attention forward kernels (attention_long.cu)
against fp32 / fp64 SDPA, their argument errors, and the model at 512x512 and 336x528 against golden vectors from the
real reference (tests/golden/hires_*, oracle/make_golden_hires.py), with the tolerance contract of test_model_gpu.py."""
import json
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests.test_hires_golden_cpu import load_hires_arrays
from tests.util import GOLDEN, rel
from vtp_b200 import lib

pytestmark = pytest.mark.gpu
BF = torch.bfloat16


def _sdpa(qkv, B, T, H, dtype=torch.float32):
    q, k, v = [t.transpose(1, 2).to(dtype) for t in qkv.view(B, T, 3, H, 64).unbind(2)]
    return F.scaled_dot_product_attention(q, k, v).transpose(1, 2).reshape(B * T, H * 64)


def _lse(qkv, B, T, H):
    q, k, _ = [t.transpose(1, 2).float() for t in qkv.view(B, T, 3, H, 64).unbind(2)]
    return torch.logsumexp(q @ k.transpose(-1, -2) * 0.125, -1)


def _run_bf16(qkv, B, T, H, prefix, with_lse):
    """out written into the middle of a NaN-filled buffer: rows the kernel must not touch sit on both sides."""
    pad = 3
    buf = torch.full((B * T + 2 * pad, H * 64), float("nan"), device="cuda", dtype=BF)
    buf[:pad] = 7.0
    buf[-pad:] = -7.0
    before = buf.clone()
    out = buf[pad:pad + B * T]
    lse = torch.full((B, H, T), float("nan"), device="cuda") if with_lse else None
    lib.attention_fwd(qkv, out, B, T, H, prefix=prefix, lse=lse)
    torch.cuda.synchronize()
    assert torch.equal(buf[:pad], before[:pad]) and torch.equal(buf[-pad:], before[-pad:])
    assert torch.isfinite(out.float()).all()
    return out, lse


@pytest.mark.parametrize("B,T,H,prefix", [(2, 258, 2, 1), (3, 386, 6, 1), (2, 577, 6, 1), (2, 694, 2, 1),
                                          (4, 1025, 16, 1), (2, 1024, 6, 0), (1, 2305, 6, 2), (1, 4097, 2, 4),
                                          (64, 1025, 6, 1)])
@pytest.mark.parametrize("with_lse", [True, False])
def test_long_attention_matches_sdpa(B, T, H, prefix, with_lse):
    g = torch.Generator(device="cuda").manual_seed(B * 1000 + T)
    qkv = (torch.randn(B * T, 3 * H * 64, device="cuda", generator=g) * 1.5).to(BF)
    out, lse = _run_bf16(qkv, B, T, H, prefix, with_lse)
    e = rel(out, _sdpa(qkv, B, T, H))
    assert e < 6e-3, e
    if with_lse:
        assert torch.isfinite(lse).all()
        el = rel(lse, _lse(qkv, B, T, H))
        assert el < 1e-4, el


def test_long_attention_online_rescale():
    """Every row's largest scores sit in the LAST key tile (logits ~ +60, earlier tiles ~ -60), so the running max
    jumps by ~120 there; for half the rows the prefix key dominates instead (logit ~ +66)."""
    B, HW, H, prefix = 2, 700, 2, 1
    T = prefix + HW
    g = torch.Generator(device="cuda").manual_seed(11)
    u = torch.zeros(64, device="cuda")
    u[0] = 1.0
    w = torch.zeros(64, device="cuda")
    w[1] = 1.0
    a = 480 ** 0.5  # q.k = 480 -> logit 480 / 8 = 60
    qkv = torch.randn(B, T, 3, H, 64, device="cuda", generator=g) * 0.3
    rows = torch.arange(T, device="cuda")
    pick_w = (rows % 2 == 1).view(1, T, 1, 1)
    qkv[:, :, 0] += torch.where(pick_w, a * w, a * u)
    last = rows >= prefix + 128 * (HW // 128)  # keys of the last (partial) tile
    qkv[:, prefix:, 1] += torch.where(last[prefix:].view(1, HW, 1, 1), a * u, -a * u)
    qkv[:, 0, 1] += 1.1 * a * w
    qkv[:, :, 2] = torch.randn(B, T, H, 64, device="cuda", generator=g)
    qkv = qkv.reshape(B * T, 3 * H * 64).to(BF)
    out, lse = _run_bf16(qkv, B, T, H, prefix, True)
    e = rel(out, _sdpa(qkv, B, T, H))
    assert e < 6e-3, e
    assert rel(lse, _lse(qkv, B, T, H)) < 1e-4


@pytest.mark.parametrize("B,T,H", [(2, 412, 3), (1, 1025, 6), (1, 1024, 2), (1, 4097, 2)])
def test_f32_tiled_attention_matches_fp64(B, T, H):
    g = torch.Generator(device="cuda").manual_seed(T)
    qkv = torch.randn(B * T, 3 * H * 64, device="cuda", generator=g) * 1.5
    out = torch.full((B * T, H * 64), float("nan"), device="cuda")
    lib.attention_fwd_f32(qkv, out, B, T, H)
    e = rel(out.double(), _sdpa(qkv, B, T, H, torch.float64))
    assert e < 1e-5, e


def test_long_attention_argument_errors():
    B, T, H = 1, 1025, 2
    qkv = torch.randn(B * T, 3 * H * 64, device="cuda").to(BF)
    out = torch.empty(B * T, H * 64, device="cuda", dtype=BF)
    with pytest.raises(lib.VtpError):
        lib.attention_fwd(qkv, out, B, T, H, prefix=1, causal=True)
    with pytest.raises(lib.VtpError):
        lib.attention_fwd(qkv, out, B, T, H, prefix=5)
    q32 = qkv.float()
    with pytest.raises(lib.VtpError):
        lib.attention_fwd_f32(q32, out.float(), B, T, H, causal=True)


# ---------------------------------------------------------------------------------------------- model level

def _load(name):
    with open(os.path.join(GOLDEN, f"hires_{name}.json")) as f:
        meta = json.load(f)
    return meta, {k: torch.from_numpy(v) for k, v in load_hires_arrays(name).items()}


def _build(name):
    from oracle.seeded import seeded_images, seeded_state_dict
    from vtp_b200.config import VTPConfig
    from vtp_b200.model import VTPModel

    meta, g = _load(name)
    m = VTPModel(VTPConfig(**meta["config"]))
    m.load_state_dict(seeded_state_dict(meta["spec"], seed=0, **meta.get("seed_opts", {})))
    x = seeded_images(meta["batch"], *meta["image_hw"])
    assert np.allclose([x.double().sum().item(), x.double().abs().sum().item()], g["x_checksum"].numpy())
    return m.cuda(), g, x.cuda(), meta


def _sub(rec, meta):
    s = meta["recon_stride"]
    return rec[..., ::s, ::s]


@pytest.mark.parametrize("name", ["tiny512", "tiny_rect", "small512"])
def test_fp32_mode_matches_reference_hires(name):
    m, g, x, meta = _build(name)
    Hi, Wi = meta["image_hw"]
    lat = m.get_reconstruction_latents(x)
    assert lat.dtype == torch.float32 and tuple(lat.shape) == (meta["batch"], 64, Hi // 16, Wi // 16)
    rec = m.get_latents_decoded_images(lat)
    assert tuple(rec.shape) == (meta["batch"], 3, Hi, Wi)
    e = {"latents": rel(lat, g["latents_fp32"]), "recon": rel(_sub(rec, meta), g["recon_fp32"]),
         "recon_from_golden_latents": rel(_sub(m.get_latents_decoded_images(g["latents_fp32"].cuda()), meta),
                                          g["recon_fp32"]),
         "img_feat": rel(m.get_clip_image_feature(x), g["img_feat_fp32"]),
         "cls": rel(m.get_last_layer_feature(x)["cls_token"], g["cls_fp32"])}
    sens = meta["ref_sensitivity_1e-6"]
    floor = dict(sens, recon_from_golden_latents=sens["recon"])
    print(name, "fp32-mode rel errors:", {k: f"{v:.2e}" for k, v in e.items()}, "ref floor:", sens)
    for k, v in e.items():
        assert v < max(1e-3, 3 * floor[k]), (k, v, floor[k])


@pytest.mark.parametrize("name", ["tiny512", "tiny_rect", "small512"])
def test_bf16_mode_matches_reference_autocast_hires(name):
    m, g, x, meta = _build(name)
    with torch.autocast("cuda", dtype=torch.bfloat16):
        lat = m.get_reconstruction_latents(x)
        assert lat.dtype == torch.bfloat16
        rec = m.get_latents_decoded_images(g["latents_bf16"].cuda().to(torch.bfloat16))
        fi = m.get_clip_image_feature(x)
        cls = m.get_last_layer_feature(x)["cls_token"]
    e, dev = {}, {}
    for key, val in (("latents", lat), ("recon", _sub(rec, meta)), ("img_feat", fi), ("cls", cls)):
        e[key] = rel(val, g[f"{key}_bf16"])
        dev[key] = (rel(val, g[f"{key}_fp32"]), rel(g[f"{key}_bf16"], g[f"{key}_fp32"]))
    print(name, "bf16-mode rel vs ref-autocast:", {k: f"{v:.2e}" for k, v in e.items()})
    print(name, "  (ours vs fp32, ref-bf16 vs fp32):", {k: (f"{a:.2e}", f"{b:.2e}") for k, (a, b) in dev.items()})
    # test_model_gpu.py's bounds, except that the absolute cap on (i) is never below d itself: at depth 12 and T = 1025
    # the chaotic cls token of the reference moves d = 3.5e-2 between its own bf16 and fp32 runs, and a fixed 2e-2 cap
    # would ask two independent bf16 evaluations to agree to 0.57 d (ours: 0.61 d, cf. 0.27-1.03 d at 256x256)
    for k, (ours, theirs) in dev.items():
        assert e[k] < min(max(2e-2, theirs), 1.25 * theirs + 2e-4), (k, e[k], theirs)
        if k == "recon":
            continue  # decoded from the reference's bf16 latents: compared with recon_bf16 above only
        assert ours < 1.15 * theirs + 2e-4, (k, ours, theirs)


def _model512():
    """the tiny512 model on a batch of two seeded 512x512 images (no reference values needed)"""
    from oracle.seeded import seeded_images

    m, _, _, meta = _build("tiny512")
    return m, seeded_images(2, 512, 512, seed=99).cuda(), meta


def test_intermediate_layers_at_512():
    m, x, meta = _model512()
    (feat,) = m.get_intermediate_layers_feature(x, n=1, reshape=True)
    assert tuple(feat.shape) == (x.shape[0], meta["config"]["vision_embed_dim"], 32, 32)
    (flat,) = m.get_intermediate_layers_feature(x, n=1, norm=True)
    assert torch.equal(flat, m.get_last_layer_feature(x)["patch_tokens"])


@pytest.mark.parametrize("autocast", [False, True])
def test_graph_replay_equals_eager_at_512(autocast):
    m, x, _ = _model512()

    def run():
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=autocast):
            lat = m.get_reconstruction_latents(x)
            return lat, m.get_latents_decoded_images(lat), m.get_clip_image_feature(x)

    eager = run()
    m.enable_cuda_graphs()
    try:
        first, again = run(), run()  # capture, then a pure replay
    finally:
        m.enable_cuda_graphs(False)
    for got in (first, again):
        for a, b in zip(got, eager):
            assert a.dtype == b.dtype and torch.equal(a, b)


def test_tokenizer_at_512():
    from vtp_b200.generation import VTP_Tokenizer

    m, x, meta = _model512()
    tok = VTP_Tokenizer(img_size=512, model=m)
    assert tok.latent_size == 32
    B = x.shape[0]
    with torch.autocast("cuda", dtype=torch.bfloat16):
        z = tok.encode_images_device(x)
        assert tuple(z.shape) == (B, 64, 32, 32)
        img = tok.decode_to_images_device(z)
        assert img.dtype == torch.uint8 and tuple(img.shape) == (B, 512, 512, 3)
        dec = m.get_latents_decoded_images(z)
    want = torch.empty_like(img)
    lib.image_to_u8(dec, tok._sub, tok._div, want)
    assert torch.equal(img, want)
