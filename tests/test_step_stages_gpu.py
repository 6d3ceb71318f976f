"""The training step's stages outside the transformer blocks, at the benchmark's shapes, against the fp64 references of
tests/stage_ref.py and tests/step_ref.py.

Pass-through spies (fixtures below) record every lib.gemm call an objective launches, and the glue kernels around
them.  Each GEMM's output is checked, per row, against gemm_ref of the very operands it received (stage_ref's header
lists the bounds); elements of the output tensor the call must not write (ldo wider than N, rows dropped or skipped by
rr_skip) must keep their old values.  Calls are named by their weight operand (the store's compute copies, the LPIPS
VGG layouts, the DINO head's weight-normed last layer) or by the gradient buffer they accumulate into; weight operands
must equal the bf16 copies of the fp32 master weights.  SwiGLU / RoPE epilogues belong to the blocks
(tests/test_block_sublayers_gpu.py) and are skipped.

Cases (VTP-Small widths, depth 1):
    lpips  LPIPSLoss.loss_and_grad on 33 images of 256² with chunk 32 (the last chunk is ragged): every conv, pool,
           tap, dgrad, pool routing and the N = 32 GEMM, each fed what the previous stage produced, every row
    rec    B = 256 at 256² with LPIPS attached: L1 / LPIPS coefficients and wiring; the LPIPS convs on the first and
           last row of every 128-row tile (the lpips case checks every row of the same code)
    clip   B = 256, world 1, text length 77: the contrastive assembly and visual_proj's dgrad into the cls rows
    ssl    B = 128, K = 65 536, head 2048 / 256, 8 local crops of 96², 30 % of the patches masked on half the global
           crops: every GEMM (tensors 65 536 wide on the first and last row of every 128-row tile), teacher / student
           row lists, t0 / t1 / row weights, the DINO student kernel on the tile rows, the DINO / iBOT loss slots
The text tower runs at the default vocabulary (49 408).  Gradient buffers are prefilled with seeded non-zero values, so
an overwrite instead of an accumulation fails.  A second run must repeat every GEMM output bit for bit, except split-K
weight gradients, and every recorded glue kernel's output.  One `STAGESTAT case | stage | k |
bound` line is printed per check.
"""
import math

import pytest
import torch

from tests import block_ref as br
from tests import stage_ref as st
from tests import step_ref as sr
from vtp_b200 import lib, lpips
from vtp_b200.config import VTPConfig
from vtp_b200.lpips import LPIPSLoss
from vtp_b200.synthetic import make_batch
from vtp_b200.train import TrainConfig, VTPTrainer

pytestmark = pytest.mark.gpu
BF = torch.bfloat16

SMALL1 = dict(vision_embed_dim=384, vision_depth=1, vision_num_heads=6, text_embed_dim=384, text_num_heads=6,
              text_depth=1, decoder_embed_dim=384, decoder_num_heads=6, decoder_depth=1)


def tile_rows(M):
    """the first and last row of every 128-row tile"""
    r = torch.cat([torch.arange(0, M, 128), torch.arange(127, M, 128), torch.tensor([M - 1])])
    return r[r < M].unique().cuda()


class Recorder:
    def __init__(self):
        self.check = True
        self.stats = {}          # stage -> [max k, bound, failure descriptions]
        self.fps = []            # fingerprints of every GEMM output, in call order
        self.gfps = []           # fingerprints of every glue kernel's output, in call order
        self.events = []         # (kernel, dict of pointers / values) in call order
        self.names = {}          # weight pointer -> (name, expected bf16 tensor)
        self.grads = {}          # gradient buffer pointer -> name
        self.sample = lambda call: False
        self.values = True       # check GEMM outputs against gemm_ref (off: wiring and names only)

    def add(self, stage, k, bound):
        k = torch.as_tensor(k).double().reshape(-1)
        m = k.max().item() if k.numel() else 0.0
        s = self.stats.setdefault(stage, [0.0, bound, []])
        s[0] = max(s[0], m) if m == m else math.inf
        if not m <= bound:
            rows = (~(k <= bound)).nonzero().flatten()
            s[2].append(f"{m:.4g} > {bound:g} in {rows.numel()} rows, first {rows[:6].tolist()} "
                        f"(128-row tiles {sorted(set((rows[:256] // 128).tolist()))[:6]})")

    def ok(self, stage, cond, what):
        self.add(stage + " " + what, 0.0 if cond else math.inf, 0.0)

    def report(self, case):
        bad = []
        for stage, (m, bound, fails) in self.stats.items():
            print(f"STAGESTAT {case} | {stage} | {m:.4g} | bound {bound:g}")
            bad += [f"{stage}: {f}" for f in fails[:3]]
        assert not bad, f"{case}:\n" + "\n".join(bad)


def _fingerprint(call):
    """two integer sums over the bits of the elements the call wrote"""
    t = call["out"]
    plain = call.get("pixel_shuffle") is None and not call.get("rr_skip") and \
        (call.get("ldo") or (t.stride(-2) if t.dim() >= 2 and call["N"] > 1 else call["N"])) == call["N"]
    idx = None if plain else st.out_index(call, st.written_rows(call)).reshape(-1)
    v = st._span(t, call["M"] * call["N"] if plain else int(idx.max()) + 1)
    v = v.view(torch.int16 if t.element_size() == 2 else torch.int32)
    v = (v if plain else v[idx]).long()
    w = torch.arange(v.numel(), device=v.device) % 65521 + 1
    return torch.stack([v.sum(), (v * w).sum()]).cpu()


def _split_k(kw):
    """a split-K GEMM: its fp32 atomics make the output order dependent"""
    return kw.get("accumulate") and kw.get("split_k", 1) != 1


GLUE_OUT = dict(lpips_prep=1, maxpool2_fwd=1, lpips_tap=3, pool_relu_bwd=3, lpips_img_grad=1, recon_l1_grad=3,
                softmax_ce=4, dino_student_ce=0, gather_rows=1)   # position of each glue kernel's output argument


@pytest.fixture
def rec(monkeypatch):
    R = Recorder()
    gemm = lib.gemm

    def spy(A, B, out, **kw):
        call = dict(kw, A=A, B=B, out=out)
        if kw.get("act", 0) in (lib.ACT_SWIGLU8, lib.ACT_ROPE) or kw.get("rope") is not None or not R.check:
            gemm(A, B, out, **kw)
            plain = kw.get("act", 0) in (lib.ACT_SWIGLU8, lib.ACT_ROPE) or kw.get("rope") is not None
            R.fps.append(None if _split_k(kw) else _fingerprint(dict(M=out.numel(), N=1, out=out) if plain else call))
            return
        before = out.clone()
        gemm(A, B, out, **kw)
        R.fps.append(None if _split_k(kw) else _fingerprint(call))
        name = _name(R, call)
        R.events.append(("gemm", dict(name=name, A=A.data_ptr(), B=B.data_ptr(), out=out.data_ptr(),
                                      mask=None if kw.get("mask_pos") is None else kw["mask_pos"].data_ptr(), call=kw)))
        if not R.values:
            return
        if kw.get("resid") is not None and kw["resid"].data_ptr() == out.data_ptr():
            call["resid"] = before           # an in-place residual: the stream as it was before the call
        rows = tile_rows(kw["M"]) if R.sample(call) else st.written_rows(call)
        for part, k in st.gemm_check(call, rows, before).items():
            R.add(f"{name} {part}", k, _bound(call, part, name))
        R.ok(name, st.untouched(call, before), "writes only its own elements")
    monkeypatch.setattr(lib, "gemm", spy)

    def wrap(name, check):
        f = getattr(lib, name)

        def s(*a, **k):
            pre = check(*a, **k) if R.check else None
            f(*a, **k)
            t = a[GLUE_OUT[name]]
            R.gfps.append(_fingerprint(dict(M=t.numel(), N=1, out=t)))
            if R.check:
                post = pre(*a, **k) if callable(pre) else None
                R.events.append((name, post if post is not None else {}))
        monkeypatch.setattr(lib, name, s)

    def prep(img, out, B, H, W, **k):
        def after(*a, **kk):
            R.add("lpips_prep", br.slack_k(out.view(-1, 32), sr.lpips_prep(img), sr.ulp_bf16(sr.lpips_prep(img)),
                                           0.0), 0.0)
            return dict(out=out.data_ptr())
        return after

    def pool(x, y, B, H, W, C, **k):
        def after(*a, **kk):
            same = (y.double() == sr.maxpool2(x)).reshape(B * H // 2 * W // 2, -1).all(1)
            R.add("maxpool2 (bit-exact)", torch.where(same, 0.0, math.inf), 0.0)
            return dict(x=x.data_ptr(), y=y.data_ptr())
        return after

    def tap(f0, f1, w, g0, P, C, coef, loss_acc, **k):
        acc0 = loss_acc.clone()

        def after(*a, **kk):
            t = sr.lpips_tap(f0.reshape(P, C), f1.reshape(P, C), w, coef)
            R.add("lpips_tap g0", br.slack_k(g0.reshape(P, C), t["g0"], sr.ulp_bf16(t["g0"]), t["g0_scale"]),
                  st.TAP_K)
            return dict(f0=f0.data_ptr(), f1=f1.data_ptr(), g0=g0.data_ptr(), loss=t["loss"].item(),
                        atomics=st.lpips_tap_atomics(P, C),
                        loss_abs=t["loss_abs"].item(), acc=loss_acc.data_ptr(), acc0=acc0)
        return after

    def prb(y, dpool, gtap, dz, B, H, W, C, **k):
        def after(*a, **kk):
            ref = sr.pool_relu_bwd(y, dpool, gtap)
            R.add("pool_relu_bwd", br.slack_k(dz.reshape(-1, C), ref.reshape(-1, C), sr.ulp_bf16(ref).reshape(-1, C),
                                              0.0), sr.LPIPS_K)
            return dict(y=y.data_ptr(), dpool=dpool.data_ptr(), gtap=None if gtap is None else gtap.data_ptr(),
                        dz=dz.data_ptr())
        return after

    def img_grad(dcol, dimg, B, H, W, **k):
        def after(*a, **kk):
            ref, sc = sr.lpips_img_grad(dcol, B, H, W)
            R.add("lpips_img_grad", br.slack_k(dimg.reshape(B * 3 * H, W), ref.reshape(-1, W), 0.0,
                                               sc.reshape(-1, W)), st.IMG_GRAD_K)
            return dict(dcol=dcol.data_ptr(), dimg=dimg.data_ptr())
        return after

    def l1(r_, tgt, dlp, out, loss_acc, B, Cc, gh, gw, r, coef, **k):
        acc0 = loss_acc.clone()

        def after(*a, **kk):
            ref, loss, labs = sr.recon_l1(r_, tgt, dlp, coef, r)
            sc = coef * torch.ones_like(ref) + (0 if dlp is None else sr.recon_l1(r_, tgt, dlp.abs(), 0.0, r)[0])
            R.add("recon_l1_grad out", br.slack_k(out, ref, sr.ulp_bf16(ref), sc), sr.ACT_K)
            R.add("loss slot 4 (L1)", sr.col_k(loss_acc.cpu() - acc0.cpu(), loss.cpu(), labs.cpu()), sr.LOSS_K)
            return dict(dlp=None if dlp is None else dlp.data_ptr(), coef=coef, numel=r_.numel(), B=B)
        return after

    def ce(logits, Rr, Cn, label0, G, coef, loss_acc, dscale_acc=None, log_scale=None, **k):
        acc0 = loss_acc.clone()

        def after(*a, **kk):
            t = sr.softmax_ce(logits, Cn, label0, coef, log_scale.item() if log_scale is not None else None)
            R.add("softmax_ce G", br.slack_k(G[:, :Cn], t["G"], sr.ulp_bf16(t["G"]), t["G_scale"]), sr.CE_K)
            return dict(label0=label0, coef=coef, loss=t["loss"].item(), loss_abs=t["loss_abs"].item(),
                        acc0=acc0.item(), acc=loss_acc)
        return after

    def student(s, tprobs, t0, t1, w, Rr, K, temp, loss_acc, **k):
        s0, acc0 = s.clone(), loss_acc.clone()

        def after(*a, **kk):
            rows = tile_rows(Rr)
            t = sr.dino_student(s0[rows], tprobs, t0[rows], None if t1 is None else t1[rows], w[rows], temp)
            R.add("dino_student_ce ds (tile rows)", br.slack_k(s[rows], t["ds"], sr.ulp_bf16(t["ds"]), t["ds_scale"]),
                  sr.DINO_K)
            loss = loss_abs = 0.0
            for r0 in range(0, Rr, 1024):             # every row, 1024 rows of fp64 [rows, K] at a time
                c = slice(r0, min(Rr, r0 + 1024))
                f = sr.dino_student(s0[c], tprobs, t0[c], None if t1 is None else t1[c], w[c], temp)
                loss, loss_abs = loss + f["loss"].item(), loss_abs + f["loss_abs"].item()
            return dict(R=Rr, t0=t0.clone(), t1=None if t1 is None else t1.clone(), w=w.clone(), loss=(loss, loss_abs),
                        acc=loss_acc.data_ptr(), d=(loss_acc - acc0).item())
        return after

    def gather(inp, out, idx, D, **k):
        return lambda *a, **kk: dict(out=out.data_ptr(), idx=idx.clone())

    for n, c in (("lpips_prep", prep), ("maxpool2_fwd", pool), ("lpips_tap", tap), ("pool_relu_bwd", prb),
                 ("lpips_img_grad", img_grad), ("recon_l1_grad", l1), ("softmax_ce", ce), ("dino_student_ce", student),
                 ("gather_rows", gather)):
        wrap(n, c)

    lp = LPIPSLoss.loss_and_grad

    def lp_spy(self, rec_, target, coef, loss_acc):
        out = lp(self, rec_, target, coef, loss_acc)
        R.events.append(("loss_and_grad", dict(coef=coef, dimg=out.data_ptr())))
        return out
    monkeypatch.setattr(LPIPSLoss, "loss_and_grad", lp_spy)
    return R


def _bound(call, part, name):
    if part == "out (GELU of out2)":
        return st.ACT_K
    if "head." in name and call["K"] >= 4096:      # the DINO head's long, same-signed reductions: see stage_ref.chain_k
        return st.chain_k(call["K"])
    if call.get("accumulate"):
        return st.WGRAD_K
    if call.get("conv") is not None:
        return st.CONV_K
    if call["N"] == 32 and call.get("b_mn") and call["K"] == 64:
        return st.DGRAD32_K
    return st.LIN_K


def _name(R, call):
    B, out = call["B"], call["out"]
    if B.data_ptr() in R.names:
        name, want = R.names[B.data_ptr()]
        R.ok(name, want is None or torch.equal(B.reshape(want.shape), want), "operand is the weights' bf16 copy")
        if name == "head.last (weight-normed)":
            R.dlogits = call["A"].data_ptr()
        return name + (" dgrad" if call.get("b_mn") and "lpips conv" not in name else "")
    if call.get("accumulate") and call["A"].data_ptr() == getattr(R, "dlogits", None):
        return "wgrad head.last (weight-normed)"
    if out.data_ptr() in R.grads and call.get("accumulate"):
        return "wgrad " + R.grads[out.data_ptr()]
    return f"gemm {call['M']}x{call['N']}x{call['K']}" + (" acc" if call.get("accumulate") else "")


def _trainer(K=512, hh=256, hb=64, n_loc=2):
    tr = VTPTrainer(VTPConfig(**SMALL1), TrainConfig(head_out_dim=K, head_hidden=hh, head_bottleneck=hb,
                                                     n_local_crops=n_loc))
    g = torch.Generator().manual_seed(5)
    s = tr.store
    for name, shape, _, _ in s.specs:
        if name == "logit_scale":
            continue
        v = s.f32(name)
        if v.dim() >= 2:
            v.copy_(torch.randn(shape, generator=g) * (1.0 / shape[-1] ** 0.5))
        elif name.endswith("_w") or name.endswith("last_g"):
            v.copy_(1 + 0.1 * torch.randn(shape, generator=g))
        else:
            v.copy_(0.05 * torch.randn(shape, generator=g))
    s.sync_compute_copies(init_teacher=True)
    return tr


def _register(R, tr):
    s = tr.store
    for name, shape, _, teacher in s.specs:
        if len(shape) == 2:
            R.names[s.bf16(name).data_ptr()] = (name, s.f32(name).to(BF))
            if teacher:
                R.names[s.tbf16(name).data_ptr()] = ("teacher " + name, s.tf32(name).to(BF))
        R.grads[s.grad(name).data_ptr()] = name
    R.names[tr.head_wn.data_ptr()] = ("head.last (weight-normed)", None)
    R.names[tr.head_wn_t.data_ptr()] = ("teacher head.last (weight-normed)", None)


def _register_lpips(R, L, vw):
    for i, w in enumerate(vw):
        R.names[L.w_fwd[i].data_ptr()] = (f"lpips conv{i}", st.w_fwd(w.cuda().float()).to(BF))
        if L.w_bwd[i] is not None:
            R.names[L.w_bwd[i].data_ptr()] = (f"lpips conv{i} dgrad", st.w_bwd(w.cuda().float()).to(BF))


def _prefill(tr):
    g = torch.Generator(device="cuda").manual_seed(77)
    tr.store.g.copy_(0.01 * torch.randn(tr.store.g.shape, device="cuda", generator=g))
    tr.loss_acc.fill_(0.25)


def _lpips_wiring(R, events, H, W):
    """walk LPIPSLoss._chunk's launches: each stage fed what the previous one produced"""
    sizes = st.lpips_sizes(H, W)
    it = iter(events)
    n_chunks = 0
    for ev in it:
        if ev[0] != "lpips_prep":
            continue
        n_chunks += 1
        feats = []
        for _ in range(2):                        # target, then reconstruction
            if feats:
                ev = next(it)
                R.ok("lpips prep", ev[0] == "lpips_prep", "order")
            x, outs = ev[1]["out"], []
            for c in st.VGG_CFG:
                ev = next(it)
                if c == "M":
                    R.ok("lpips maxpool2", ev[0] == "maxpool2_fwd" and ev[1]["x"] == x, "fed the conv output")
                    x = ev[1]["y"]
                    continue
                i = len(outs)
                R.ok(f"lpips conv{i}", ev[0] == "gemm" and ev[1]["A"] == x and ev[1]["name"] == f"lpips conv{i}",
                     "fed the previous stage")
                x = ev[1]["out"]
                outs.append(x)
            feats.append(outs)
        a1, a0 = feats
        gt = {}
        for k, ti in enumerate(st.TAPS):
            ev = next(it)
            R.ok(f"lpips tap {k}", ev[0] == "lpips_tap" and ev[1]["f0"] == a0[ti] and ev[1]["f1"] == a1[ti],
                 "fed conv outputs of reconstruction and target")
            gt[ti] = ev[1]["g0"]
        dz = gt[12]
        for i in range(12, 0, -1):
            ev = next(it)
            pooled = sizes[i - 1] != sizes[i]
            R.ok(f"lpips conv{i} dgrad", ev[0] == "gemm" and ev[1]["A"] == dz and ev[1]["name"] == f"lpips conv{i} dgrad"
                 and ev[1]["mask"] == (None if pooled else a0[i - 1]), "fed dz, masked by the producer's ReLU")
            dz = ev[1]["out"]
            if pooled:
                ev = next(it)
                R.ok(f"pool_relu_bwd into conv{i - 1}", ev[0] == "pool_relu_bwd" and ev[1]["y"] == a0[i - 1]
                     and ev[1]["dpool"] == dz and ev[1]["gtap"] == gt.get(i - 1),
                     "fed the dgrad, the conv output and that conv's tap gradient")
                dz = ev[1]["dz"]
        ev = next(it)
        R.ok("lpips conv0 (N = 32 dgrad)", ev[0] == "gemm" and ev[1]["A"] == dz and ev[1]["name"] == "lpips conv0",
             "fed dz of conv0")
        dcol = ev[1]["out"]
        ev = next(it)
        R.ok("lpips_img_grad", ev[0] == "lpips_img_grad" and ev[1]["dcol"] == dcol, "fed the N = 32 dgrad")
    return n_chunks


def _second_run(R, fn):
    fps, gfps = R.fps, R.gfps
    R.check, R.fps, R.gfps, R.events = False, [], [], []
    fn()
    torch.cuda.synchronize()
    diff = [i for i, (a, b) in enumerate(zip(fps, R.fps)) if a is not None and not torch.equal(a, b)]
    R.ok("every GEMM output but split-K", len(fps) == len(R.fps) and not diff, f"bit-identical on a second run {diff[:5]}")
    diff = [i for i, (a, b) in enumerate(zip(gfps, R.gfps)) if not torch.equal(a, b)]
    R.ok("every glue kernel output", len(gfps) == len(R.gfps) and not diff, f"bit-identical on a second run {diff[:5]}")


# --------------------------------------------------------------------------------------------------------------- cases

def test_lpips_chain(rec):
    vw, vb, lw = lpips.random_weights(0)
    L = LPIPSLoss(vw, vb, lw, chunk=32)
    _register_lpips(rec, L, vw)
    g = torch.Generator(device="cuda").manual_seed(3)
    x = torch.rand(33, 3, 256, 256, device="cuda", generator=g)
    y = (x + 0.1 * torch.randn(x.shape, device="cuda", generator=g)).clamp(0, 1)
    acc = torch.full((1,), 0.25, device="cuda")
    dimg = L.loss_and_grad(y, x, 0.03, acc)
    torch.cuda.synchronize()
    events = list(rec.events)
    rec.ok("lpips", _lpips_wiring(rec, events, 256, 256) == 2, "two chunks (32 + 1 images)")
    igs = [e[1]["dimg"] for e in events if e[0] == "lpips_img_grad"]
    rec.ok("lpips_img_grad", igs == [dimg.data_ptr(), dimg[32:].data_ptr()], "writes each chunk's slice of dimg")
    taps = [e[1] for e in events if e[0] == "lpips_tap"]
    loss = sum(t["loss"] for t in taps)
    rec.add("loss (lpips slot)", sr.col_k(acc.cpu() - 0.25, torch.tensor([loss]), torch.tensor(
        [sum(t["loss_abs"] for t in taps)])), st.lpips_loss_k(taps))
    out1 = dimg.clone()
    _second_run(rec, lambda: L.loss_and_grad(y, x, 0.03, acc))
    rec.report("lpips")
    # a shape the VGG stack cannot take is refused before any launch
    before = acc.clone()
    with pytest.raises(ValueError, match="LPIPS"):
        L.loss_and_grad(y[:, :, :200, :200].contiguous(), x[:, :, :200, :200].contiguous(), 0.03, acc)
    torch.cuda.synchronize()
    assert torch.equal(acc, before)
    assert out1.isfinite().all()


def test_rec_stages(rec):
    tr = _trainer()
    vw, vb, lw = lpips.random_weights(0)
    L = tr.enable_lpips(LPIPSLoss(vw, vb, lw, chunk=32))
    _register(rec, tr)
    _register_lpips(rec, L, vw)
    rec.sample = lambda call: call.get("conv") is not None or call["N"] == 32 and call["K"] == 64
    img = make_batch(256)["rec_image"].cuda().clamp(-1, 1)
    _prefill(tr)
    tr.rec_fwd_bwd(img, 0.8)
    torch.cuda.synchronize()
    ev = rec.events
    lps = [e[1] for e in ev if e[0] == "loss_and_grad"]
    l1s = [e[1] for e in ev if e[0] == "recon_l1_grad"]
    c1, c2 = st.recon_coefs(img.numel(), 256, 256, 0.8, tr.tc.lpips_weight)
    rec.ok("rec LPIPS", len(lps) == 1 and lps[0]["coef"] == c2, "coefficient weight·lpips_weight/nB")
    rec.ok("recon_l1_grad", len(l1s) == 1 and l1s[0]["coef"] == c1, "coefficient weight/(numel/B·nB)")
    rec.ok("recon_l1_grad", l1s[0]["dlp"] == lps[0]["dimg"], "adds the LPIPS image gradient")
    taps = [e[1] for e in ev if e[0] == "lpips_tap"]
    rec.add("loss slot 5 (LPIPS)", sr.col_k(tr.loss_acc[5:6].cpu() - 0.25, torch.tensor([sum(t["loss"] for t in taps)]),
                                           torch.tensor([sum(t["loss_abs"] for t in taps)])), st.lpips_loss_k(taps))
    names = {e[1]["name"] for e in ev if e[0] == "gemm"}
    for want in ("trunk.bneck.w", "decoder.proj_in.w", "decoder.proj_out.w", "trunk.bneck.w dgrad",
                 "decoder.proj_in.w dgrad", "wgrad trunk.bneck.w", "wgrad decoder.proj_in.w", "wgrad trunk.patch.w"):
        rec.ok(want, want in names, "launched")
    _prefill(tr)
    _second_run(rec, lambda: tr.rec_fwd_bwd(img, 0.8))
    rec.report("rec")


def test_clip_stages(rec):
    tr = _trainer()
    _register(rec, tr)
    b = make_batch(256)
    _prefill(tr)
    tr.clip_fwd_bwd(b["image"].cuda(), b["text"].cuda(), 1.0)
    torch.cuda.synchronize()
    ev = rec.events
    ces = [e[1] for e in ev if e[0] == "softmax_ce"]
    rec.ok("softmax_ce", len(ces) == 2 and all(c["label0"] == 0 and c["coef"] == 0.5 / 256 for c in ces),
           "labels rank·B + r, coef 0.5/B, both directions")
    rec.add("loss slot 0 (contrastive)", sr.col_k(tr.loss_acc[0:1].cpu() - 0.25, torch.tensor(
        [sum(c["loss"] for c in ces)]), torch.tensor([0.25 + sum(c["loss_abs"] for c in ces)])), st.CE_LOSS_K)
    vp = [e[1] for e in ev if e[0] == "gemm" and e[1]["name"] == "visual_proj.w dgrad"]
    rec.ok("visual_proj.w dgrad", len(vp) == 1 and vp[0]["call"].get("ldo") == 257 * 384,
           "lands on the cls rows (ldo = T·D)")
    cross = [e[1] for e in ev if e[0] == "gemm" and e[1]["call"].get("a_mn") and e[1]["call"]["K"] == 256
             and e[1]["call"].get("accumulate") and e[1]["call"]["M"] == 256]
    rec.ok("contrastive cross terms", len(cross) == 2, "accumulate into dfi / dft")
    _prefill(tr)
    _second_run(rec, lambda: tr.clip_fwd_bwd(b["image"].cuda(), b["text"].cuda(), 1.0))
    rec.report("clip")


def test_ssl_stages(rec):
    B, n_loc = 128, 8
    tr = _trainer(K=65536, hh=2048, hb=256, n_loc=n_loc)
    _register(rec, tr)
    b = make_batch(B)
    gc, lc = b["global_crops"].cuda(), b["local_crops"].cuda()
    mi, mw = b["mask_indices"].cuda(), b["masks_weight"].cuda()
    rec.sample = lambda call: call["N"] >= 65536 or call["K"] >= 65536 or call["M"] >= 65536   # 65 536-wide tensors
    _prefill(tr)
    centres = tr.center_dino.clone(), tr.center_ibot.clone()   # the step's EMA moves them; the second run restores
    tr.ssl_fwd_bwd(gc, lc, mi, mw, 0.9)
    torch.cuda.synchronize()
    ev = rec.events
    T, HW = 257, 256
    L = st.ssl_lists(B, n_loc, T, HW, mi, mw, 0.9, B)
    gem = [e[1] for e in ev if e[0] == "gemm"]
    t_in = [g["A"] for g in gem if g["name"] == "teacher head.mlp0.w"]
    s_in = [g["A"] for g in gem if g["name"] == "head.mlp0.w"]
    gathers = {e[1]["out"]: e[1]["idx"] for e in ev if e[0] == "gather_rows"}
    rec.ok("teacher head input", len(t_in) == 1 and t_in[0] in gathers
           and torch.equal(gathers[t_in[0]].long(), L["teacher_rows"]), "rows: swapped cls, then masked patches")
    sg = None if not s_in else s_in[0] + n_loc * B * 384 * 2
    rec.ok("student head input", sg in gathers and torch.equal(gathers[sg].long(), L["student_rows"]),
           "global rows: cls, then masked patches")
    sts = {e[1]["acc"]: e[1] for e in ev if e[0] == "dino_student_ce"}   # by the loss slot each launch adds into
    nl, B2, n_m = n_loc * B, 2 * B, mi.numel()
    for nm, (r0, r1), slot in (("local", (0, nl), 1), ("global", (nl, nl + B2), 2), ("ibot", (nl + B2, nl + B2 + n_m), 3)):
        s = sts.get(tr.loss_acc[slot:slot + 1].data_ptr())
        good = s is not None and s["R"] == r1 - r0 and torch.equal(s["t0"], L["t0"][r0:r1]) and \
            torch.equal(s["t1"], L["t1"][r0:r1]) and torch.allclose(s["w"].double(), L["wrow"][r0:r1], rtol=1e-7, atol=0)
        rec.ok(f"dino_student_ce {nm}", good, "t0 / t1 / row weights")
        if s is not None:
            rec.add(f"loss slot {slot} ({nm})", sr.col_k(torch.tensor([s["d"]]), torch.tensor([s["loss"][0]]),
                                                         torch.tensor([s["loss"][1]])), sr.LOSS_K)
    _prefill(tr)
    tr.center_dino.copy_(centres[0]), tr.center_ibot.copy_(centres[1])
    _second_run(rec, lambda: tr.ssl_fwd_bwd(gc, lc, mi, mw, 0.9))
    rec.report("ssl")
