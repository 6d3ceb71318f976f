"""Training above 256x256: the hand-written step (vtp_b200/train.py) at 512x512 (HW = 1024 patch tokens) and 336x528
(21 x 33 = 693, so a ragged key tile reads the next image's rows) against autograd on the CPU oracle, with the tiny
config of tests/test_train_gpu.py.  Every trunk and decoder attention backward here runs the streaming kernels
(vtp_attention_bwd_long); the SSL case also runs the packed single-pass kernel on its local crops in the same step.

Gradients are compared per tensor under the bound of tests/test_train_gpu.py::_check: max(4 %, 1.5 x |oracle bf16 -
oracle fp32|) where the fp32 oracle is run, the flat 6 % otherwise (the SSL and stochastic-depth cases, as at 256²).
"""
import pytest
import torch

from oracle import vtp_oracle as vo
from oracle.seeded import seeded_captions, seeded_images
from tests import test_train_gpu as tt
from tests.util import rel

pytestmark = pytest.mark.gpu

GEOMS = {"sq512": (512, 512), "rect336x528": (336, 528)}


def _setup(hw):
    c = tt._setup("tiny")
    c.h, c.w = hw
    c.HW = (c.h // 16) * (c.w // 16)
    return c


@pytest.mark.parametrize("geom", list(GEOMS))
def test_rec_objective_gradients_hires(geom):
    c = _setup(GEOMS[geom])
    tr = c.tr
    x = seeded_images(2, c.h, c.w)

    def oracle(mode):
        q = tt._leafs(c.sd)
        lat = vo.reconstruction_latents(x, q, depth=2, heads=c.heads, mode=mode)
        rec_ = vo.decode_latents(lat, q, depth=2, heads=c.dheads, mode=mode)
        l = vo.recon_loss(rec_, x, None)
        l.backward()
        return q, rec_.detach(), l

    p, rec, loss = oracle("bf16")
    p32, _, _ = oracle("fp32")
    out = tr.rec_fwd_bwd(x.cuda(), 1.0, return_image=True)
    torch.cuda.synchronize()
    assert rel(out, rec) < 2e-2
    assert abs(tr.loss_acc[4].item() - loss.item()) < tt.TOL_L * loss.item()
    tt.FLOORS.clear()
    g, g32 = (lambda k: p[k].grad), (lambda k: p32[k].grad)
    tt._vit_checks(tr, p, "trunk.", "trunk.", [0, 1], False, p32)
    tt._vit_checks(tr, p, "pixel_decoder.", "decoder.", [0, 1], True, p32)
    for ours, key, flat in (("trunk.patch.w", "trunk.patch_embed.proj.weight", True),
                            ("trunk.cls", "trunk.cls_token", False), ("trunk.bneck.w", "trunk.feature_bottleneck.weight", False),
                            ("decoder.proj_in.w", "pixel_decoder.proj_in.weight", True),
                            ("decoder.proj_out.w", "pixel_decoder.proj_out.weight", True)):
        tt._check(tr, ours, g(key).flatten(1) if flat else g(key), g32(key).flatten(1) if flat else g32(key))
    tt._summary(geom, "rec")


def test_rec_objective_with_lpips_gradients_512():
    """L1 + LPIPS (frozen seeded-random VGG16) on one 512² image"""
    from vtp_b200.lpips import LPIPSLoss, random_weights

    c = _setup(GEOMS["sq512"])
    tr = c.tr
    vw, vb, lw = random_weights(0)
    tr.enable_lpips(LPIPSLoss(vw, vb, lw, device="cuda", chunk=1))
    x = seeded_images(1, 512, 512) * 0.5
    p = tt._leafs(c.sd)
    lat = vo.reconstruction_latents(x, p, depth=2, heads=c.heads, mode="bf16")
    rec = vo.decode_latents(lat, p, depth=2, heads=c.dheads, mode="bf16")
    lp = vo.lpips(rec, x, vw, vb, lw, mode="bf16")
    loss = vo.recon_loss(rec, x, lp, 1.0)
    loss.backward()
    tr.rec_fwd_bwd(x.cuda(), 1.0)
    torch.cuda.synchronize()
    l1, lpv = tr.loss_acc[4].item(), tr.loss_acc[5].item()
    assert abs(lpv - lp.mean().item()) < 3e-2 * abs(lp.mean().item()), (lpv, lp.mean().item())
    assert abs(l1 + lpv - loss.item()) < tt.TOL_L * loss.item()
    tt.FLOORS.clear()
    tt._vit_checks(tr, p, "pixel_decoder.", "decoder.", [0, 1], True)
    tt._vit_checks(tr, p, "trunk.", "trunk.", [0, 1], False)
    tt._check(tr, "decoder.proj_out.w", p["pixel_decoder.proj_out.weight"].grad.flatten(1))
    tt._check(tr, "trunk.bneck.w", p["trunk.feature_bottleneck.weight"].grad)
    tt._summary("sq512", "rec+lpips")


@pytest.mark.parametrize("geom", list(GEOMS))
def test_clip_objective_gradients_hires(geom):
    c = _setup(GEOMS[geom])
    tr = c.tr
    B = 3
    x = seeded_images(B, c.h, c.w)
    ids = seeded_captions(B, 77, c.vocab)

    def oracle(mode):
        q = tt._leafs(c.sd)
        fi = vo.clip_image_feature(x, q, depth=2, heads=c.heads, mode=mode)
        ft = vo.text_feature(ids, q, layers=2, heads=c.theads, mode=mode)
        l = vo.clip_loss(vo._r(fi, mode), vo._r(ft, mode), q["logit_scale"].exp())
        l.backward()
        return q, l

    p, loss = oracle("bf16")
    p32, _ = oracle("fp32")
    tr.clip_fwd_bwd(x.cuda(), ids.cuda(), 1.0)
    torch.cuda.synchronize()
    assert abs(tr.loss_acc[0].item() - loss.item()) < tt.TOL_L * abs(loss.item()), (tr.loss_acc[0].item(), loss.item())
    tt.FLOORS.clear()
    g, g32 = (lambda k: p[k].grad), (lambda k: p32[k].grad)
    tt._vit_checks(tr, p, "trunk.", "trunk.", [0, 1], False, p32)
    tt._check(tr, "visual_proj.w", g("visual_proj.weight"), g32("visual_proj.weight"))
    tt._check(tr, "trunk.patch.w", g("trunk.patch_embed.proj.weight").flatten(1),
              g32("trunk.patch_embed.proj.weight").flatten(1))
    tt._check(tr, "trunk.cls", g("trunk.cls_token"), g32("trunk.cls_token"))
    tt._summary(geom, "clip")


@pytest.mark.parametrize("geom", list(GEOMS))
def test_ssl_objective_gradients_hires(geom):
    """global crops at the high resolution (streaming backward), local crops of 112² (T = 50: packed single-pass
    backward), both in the same step"""
    c = _setup(GEOMS[geom])
    tr, sd, hsd, K = c.tr, c.sd, c.hsd, c.K
    B, n_loc, local = 2, 2, 112
    gc = seeded_images(2 * B, c.h, c.w, seed=11)
    lc = seeded_images(n_loc * B, local, local, seed=12)
    HW = c.HW
    gsel = torch.Generator().manual_seed(5)
    masks = torch.zeros(2 * B, HW, dtype=torch.bool)
    for img in (0, 3):
        masks[img, torch.randperm(HW, generator=gsel)[:int(0.3 * HW)]] = True
    mask_idx = masks.flatten().nonzero().flatten()
    mw = (1.0 / masks.sum(-1).clamp(min=1).float())[:, None].expand_as(masks)[masks]
    p = tt._leafs(sd)
    hp = tt._leafs(hsd)
    hp_full = {"h." + k: v for k, v in hp.items()}
    with torch.no_grad():
        t_out = vo.trunk_forward([gc], [None], sd, depth=2, heads=c.heads, mode="bf16", use_bottleneck=False)[0]
        tcls = t_out["x_norm_clstoken"]
        tcls = torch.cat([tcls[B:], tcls[:B]])
        tpatch = t_out["x_norm_patchtokens"].flatten(0, 1)[mask_idx]
        th = {"h." + k: v for k, v in hsd.items()}
        tlog = vo.dino_head(vo._r(torch.cat([tcls, tpatch]), "bf16"), th, "h.", mode="bf16")
        tp_cls = vo.teacher_probs(tlog[:2 * B], torch.zeros(K), 0.07)
        tp_m = vo.teacher_probs(tlog[2 * B:], torch.zeros(K), 0.07)
    sg, sl = vo.trunk_forward([gc, lc], [masks, None], p, depth=2, heads=c.heads, mode="bf16", use_bottleneck=False)
    s_in = torch.cat([sl["x_norm_clstoken"], sg["x_norm_clstoken"], sg["x_norm_patchtokens"].flatten(0, 1)[mask_idx]])
    slog = vo.dino_head(vo._r(s_in, "bf16"), hp_full, "h.", mode="bf16")
    nl = n_loc * B
    terms = vo.dino_ibot_loss(slog[:nl], slog[nl:nl + 2 * B], slog[nl + 2 * B:], tp_cls, tp_m, mw, n_local=n_loc,
                              n_images=2 * B)
    loss = terms["dino_local"] + terms["dino_global"] + terms["ibot"]
    loss.backward()
    tr.ssl_fwd_bwd(gc.cuda(), lc.cuda(), mask_idx.cuda(), mw.cuda(), 1.0)
    torch.cuda.synchronize()
    got = tr.loss_acc[1:4].cpu()
    for j, k in enumerate(("dino_local", "dino_global", "ibot")):
        assert abs(got[j].item() - terms[k].item()) < 3e-2 * abs(terms[k].item()), (k, got[j].item(), terms[k].item())
    tt.FLOORS.clear()
    tt._vit_checks(tr, p, "trunk.", "trunk.", [0, 1], False)
    tt._check(tr, "trunk.patch.w", p["trunk.patch_embed.proj.weight"].grad.flatten(1))
    tt._check(tr, "trunk.cls", p["trunk.cls_token"].grad)
    tt._check(tr, "trunk.mask_token", p["trunk.mask_token"].grad)
    for j in (0, 2, 4):
        tt._check(tr, f"head.mlp{j}.w", hp[f"mlp.{j}.weight"].grad)
    tt._summary(geom, "ssl")


def test_stochastic_depth_gradients_512():
    """reconstruction with rec_drop_rate 0.5 and preset subsets: the attention backward runs on the kept images only"""
    c = _setup(GEOMS["sq512"])
    tr = c.tr
    B, ratio = 4, 0.5
    x = seeded_images(B, 512, 512)
    keep = max(int(B * (1 - ratio)), 1)
    gen = torch.Generator().manual_seed(77)
    presets = [torch.randperm(B, generator=gen)[:keep] for _ in range(4)]
    sc = B / keep
    p = tt._leafs(c.sd)
    drops = [[(presets[0], sc, presets[1], sc), (presets[2], sc, presets[3], sc)]]
    o = vo.trunk_forward([x], [None], p, depth=2, heads=c.heads, mode="bf16", drops=drops)[0]
    pt = o["x_norm_patchtokens"]
    lat = pt.transpose(1, 2).reshape(B, pt.shape[-1], 32, 32)
    rec = vo.decode_latents(lat, p, depth=2, heads=c.dheads, mode="bf16")
    loss = vo.recon_loss(rec, x, None)
    loss.backward()
    tr.tc.rec_drop_rate = ratio
    tr.drop_presets = [presets]
    out = tr.rec_fwd_bwd(x.cuda(), 1.0, return_image=True)
    torch.cuda.synchronize()
    assert rel(out, rec.detach()) < 2e-2
    assert abs(tr.loss_acc[4].item() - loss.item()) < tt.TOL_L * loss.item()
    tt.FLOORS.clear()
    tt._vit_checks(tr, p, "trunk.", "trunk.", [0, 1], False)
    tt._vit_checks(tr, p, "pixel_decoder.", "decoder.", [0, 1], True)
    tt._check(tr, "trunk.patch.w", p["trunk.patch_embed.proj.weight"].grad.flatten(1))
    tt._check(tr, "trunk.cls", p["trunk.cls_token"].grad)
    tt._summary("sq512", "stochastic depth rec")


def _batch512(B=4, n_loc=2, seed=0):
    HW = 1024
    masks = torch.zeros(2 * B, HW, dtype=torch.bool)
    masks[::2, :300] = True
    return dict(image=seeded_images(B, 512, 512, seed=seed + 1).cuda(), text=seeded_captions(B, 77, 1000).cuda(),
                global_crops=seeded_images(2 * B, 512, 512, seed=seed + 21).cuda(),
                local_crops=seeded_images(n_loc * B, 112, 112, seed=seed + 22).cuda(),
                mask_indices=masks.flatten().nonzero().flatten().cuda(),
                masks_weight=(1.0 / masks.sum(-1).clamp(min=1).float())[:, None].expand_as(masks)[masks].cuda(),
                rec_image=seeded_images(B, 512, 512, seed=seed + 3).cuda())


def test_graph_step_equals_eager_steps_512():
    """the captured step (3 objectives + LPIPS + optimiser + EMA) at 512² replays like eager launches, to the tolerance
    of test_train_gpu.py::test_graph_step_equals_eager_steps (the δ workspace is allocated inside the graph).  The
    learning rate is 5e-5 rather than 2e-4: at 512² the split-K weight-gradient sums run over 16x more tokens, and at
    2e-4 the contrastive loss of these 4 images falls to ~0.02 by step 5, where two EAGER runs already differ by 8e-4
    relative through the reordered fp32 atomics alone (measured on an H100)."""
    batch = _batch512()
    b2 = dict(batch)
    b2["rec_image"] = seeded_images(4, 512, 512, seed=77).cuda()
    seq = [batch, batch, b2, batch, b2]

    def trainer():
        t = tt._setup("tiny").tr
        t.hyper[3] = 5e-5
        t.enable_lpips(seed=0, chunk=2)
        return t

    te = trainer()
    le = [te.train_step(b).cpu().clone() for b in seq]
    tg = trainer()
    tg.capture_step(batch, warmup=2)
    lg = [tg.replay_step(b).cpu().clone() for b in seq[2:]]
    assert tg.step_count == te.step_count == 5
    for a, b in zip(le[2:], lg):
        assert torch.isfinite(b).all()
        assert torch.allclose(a, b, rtol=2e-3, atol=1e-5), (a, b)
    assert rel(tg.store.p, te.store.p) < 1e-4
    assert rel(tg.store.tp, te.store.tp) < 1e-5


def test_pipeline_feeds_hires_steps_and_learns():
    """TrainBatchPipeline at image_size 512 / local_size 192 feeding train_step: losses finite, the reconstruction L1
    (rec_image is the whole source image resized, the same every step) goes down"""
    from vtp_b200.data import TrainBatchPipeline

    tr = tt._setup("tiny").tr
    tr.hyper[3] = 2e-4
    B = 2
    src = (torch.rand(B, 600, 640, 3, generator=torch.Generator().manual_seed(3)) * 255).to(torch.uint8)
    ids = seeded_captions(B, 77, 1000)
    pipe = TrainBatchPipeline("cuda", image_size=512, local_size=192, n_local=2, seed=1)
    pipe.submit(src, ids)
    hist = []
    for _ in range(6):
        batch = pipe.get()
        pipe.submit(src, ids)
        assert batch["global_crops"].shape == (2 * B, 3, 512, 512) and batch["local_crops"].shape == (2 * B, 3, 192, 192)
        hist.append(tr.train_step(batch).cpu().clone())
    pipe.get()
    pipe.close()
    assert all(torch.isfinite(h).all() for h in hist)
    assert hist[-1][4] < hist[0][4]
    assert hist[-1][0] < hist[0][0] + 1e-3
