"""Zero-shot classification on the device (vtp_b200/zero_shot.py, csrc/zero_shot.cu).

Kernels against fp64 / exact restatements, the bucketed text encoding against the full 77-token tower (bit-identical),
parity with the reference's own golden run (tests/golden/zero_shot_tiny.*), the evaluator's graph / dtype / sync
behaviour and the command line end to end."""
import json
import os
import re

import numpy as np
import pytest
import torch

from oracle.seeded import seeded_images, seeded_state_dict
from tests.test_zero_shot_cpu import GOLDEN, prompt_fixture, rank_rule
from vtp_b200 import lib
from vtp_b200 import zero_shot as Z
from vtp_b200.config import VTPConfig, preset
from vtp_b200.model import VTPModel

pytestmark = pytest.mark.gpu
U = 2.0 ** -24


def _model(cfg, seed=0):
    m = VTPModel(cfg)
    m.load_state_dict(seeded_state_dict({k: list(v.shape) for k, v in m.state_dict().items()}, seed=seed))
    return m.cuda().eval()


# ------------------------------------------------------------------------------------------------ vtp_zs_class_embed
def _class_embed_ref(feat64: torch.Tensor, C: int, T: int):
    """fp64: f = x / max(|x|, eps); mean over t; normalise.  Also the summed magnitudes of the template mean."""
    x = feat64.view(C, T, -1)
    f = x / x.norm(dim=-1, keepdim=True).clamp_min(1e-12)
    m = f.mean(1)
    n = m.norm(dim=-1, keepdim=True).clamp_min(1e-12)
    return m / n, f.abs().mean(1) / n


@pytest.mark.parametrize("C", [1, 37, 1000])
@pytest.mark.parametrize("T", [1, 80])
@pytest.mark.parametrize("Ed", [384, 512, 768, 1024])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("permuted", [False, True])
def test_class_embed_against_fp64(C, T, Ed, dtype, permuted):
    g = torch.Generator().manual_seed(C * 7 + T + Ed)
    x = (torch.randn(C * T, Ed, generator=g) * 0.3 + 0.05 * torch.randn(C, 1, Ed, generator=g).repeat_interleave(T, 0)
         .view(C * T, Ed)).to(dtype)
    x[0] = 0                                              # a zero feature: clamp_min(eps) keeps it 0
    Cp = (C + 7) // 8 * 8
    out = torch.full((Cp, Ed), float("nan"), device="cuda")
    if permuted:
        perm = torch.randperm(C * T, generator=g)
        buf = torch.empty_like(x)
        buf[perm] = x                                     # prompt p lives at row perm[p]
        lib.zs_class_embed(buf.cuda(), out, C, T, row_of=perm.to(torch.int32).cuda())
    else:
        lib.zs_class_embed(x.cuda(), out, C, T)
    ref, mag = _class_embed_ref(x.double(), C, T)
    got = out.cpu().double()
    assert torch.equal(got[C:], torch.zeros(Cp - C, Ed, dtype=torch.float64))
    # a few fp32 ulps per term, scaled by the summed magnitudes (tests/step_ref.py's rule) plus the two norms' sums
    bound = 8 * U * (mag + got[:C].abs()) * (Ed ** 0.5 + 4) + 4 * U * got[:C].abs()
    err = (got[:C] - ref).abs()
    assert (err <= bound).all(), float((err / bound.clamp_min(1e-30)).max())
    again = torch.empty_like(out)
    if permuted:
        lib.zs_class_embed(buf.cuda(), again, C, T, row_of=perm.to(torch.int32).cuda())
    else:
        lib.zs_class_embed(x.cuda(), again, C, T)
    assert torch.equal(again, out)


def test_image_operand_rounding():
    g = torch.Generator().manual_seed(3)
    for xd in (torch.float32, torch.bfloat16):
        x = (torch.randn(300, 768, generator=g) * 2).to(xd).cuda()
        x[5] = 0
        n = x.float().double().norm(dim=-1, keepdim=True).clamp_min(1e-12)
        ref = 100.0 * (x.double() / n)
        for od in (torch.float32, torch.bfloat16):
            a = torch.empty(300, 768, dtype=od, device="cuda")
            lib.zs_image_operand(x, a, 100.0)
            got = a.double()
            if od == torch.float32:
                assert ((got - ref).abs() <= 40 * U * ref.abs() + 1e-30).all()
            else:                                      # one bf16 rounding of the fp32 value (ulp 2^-8 relative)
                assert ((got - ref).abs() <= (2.0 ** -8 + 40 * U) * ref.abs() + 1e-30).all()
            assert (got[5] == 0).all()


# ------------------------------------------------------------------------------------------------ vtp_zs_rank
def _rank_case(B, C, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    logits = torch.randn(B, C, generator=g) * 10
    if dtype == torch.bfloat16:
        logits = (logits / 2).round() * 2 + 20          # many exact ties near 20-30
    logits = logits.to(dtype)
    targets = torch.randint(0, C, (B,), generator=g)
    nan_rows = torch.randperm(B, generator=g)[: max(1, B // 16)]
    for i, r in enumerate(nan_rows.tolist()):
        logits[r, torch.randint(0, C, (1 + i % 3,), generator=g)] = float("nan")
        if i % 4 == 0:
            logits[r, targets[r]] = float("nan")        # NaN target logit
    bad = torch.randperm(B, generator=g)[: max(1, B // 32)]
    targets[bad[::2]] = -1
    targets[bad[1::2]] = C + 3
    return logits, targets


@pytest.mark.parametrize("B,C", [(1, 1), (7, 37), (128, 1000), (4096, 1000), (513, 999)])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_rank_exact(B, C, dtype):
    logits, targets = _rank_case(B, C, dtype, B + C)
    ld = (C + 7) // 8 * 8 + 8
    buf = torch.full((B, ld), float("inf"), dtype=dtype)   # columns past C must be ignored
    buf[:, :C] = logits
    ranks = torch.full((B,), -7, dtype=torch.int32, device="cuda")
    counts = torch.tensor([5, 0, 0], dtype=torch.int64, device="cuda")
    lib.zs_rank(buf.cuda(), C, targets.cuda(), ranks, counts, ks=(1, 5, 10))
    ref = rank_rule(logits.float().numpy(), targets.numpy())
    assert np.array_equal(ranks.cpu().numpy(), ref)
    assert counts.cpu().tolist() == [5 + int((ref < 1).sum()), int((ref < 5).sum()), int((ref < 10).sum())]


# ------------------------------------------------------------------------------------------------ bucketed text encoding
@pytest.fixture(scope="module")
def fixture_ids():
    return prompt_fixture()


@pytest.mark.parametrize("mode", ["fp32", "bf16"])
def test_bucketed_text_features_bit_identical_tiny(fixture_ids, mode):
    _, ids = fixture_ids
    m = _model(preset("tiny", text_vocab_size=49408))
    m.compute_mode = mode
    feats, row_of = Z.encode_prompts(m, ids, mode)
    for s in range(0, len(ids), 8000):
        full = m.get_clip_text_feature(ids[s:s + 8000].cuda(), normalize=False)
        assert torch.equal(feats[torch.from_numpy(row_of[s:s + 8000]).long().cuda()], full), s


@pytest.mark.parametrize("mode", ["fp32", "bf16"])
def test_bucketed_text_features_bit_identical_wide(fixture_ids, mode):
    _, ids = fixture_ids
    cfg = preset("tiny", text_embed_dim=768, text_num_heads=12, text_depth=2, text_vocab_size=49408)
    m = _model(cfg, seed=1)
    m.compute_mode = mode
    sub = torch.cat([ids[:2400], ids[-800:]])            # the first 30 classes and the last 10
    feats, row_of = Z.encode_prompts(m, sub, mode, max_rows=1000)
    full = m.get_clip_text_feature(sub.cuda(), normalize=False)
    assert torch.equal(feats[torch.from_numpy(row_of).long().cuda()], full)


# ------------------------------------------------------------------------------------------------ golden parity
def _golden():
    with open(os.path.join(GOLDEN, "zero_shot_tiny.json")) as f:
        meta = json.load(f)
    return meta, np.load(os.path.join(GOLDEN, "zero_shot_tiny.npz"))


class _FixtureTokenizer:
    """list[str] -> the reference tokenizer's ids, read from the prompts fixture (no vocabulary needed)."""

    def __init__(self, meta, ids):
        texts = [t.format(c=c) for c in meta["classnames"] for t in meta["templates"]]
        self.row = {s: i for i, s in enumerate(texts)}
        self.ids = ids

    def __call__(self, texts):
        return self.ids[[self.row[s] for s in texts]]


@pytest.fixture(scope="module")
def golden_model():
    meta, z = _golden()
    m = VTPModel(VTPConfig(**meta["config"]))
    m.load_state_dict(seeded_state_dict(meta["spec"], seed=meta["seed"]))
    return m.cuda().eval()


@pytest.mark.parametrize("mode", ["fp32", "bf16"])
def test_golden_parity(fixture_ids, golden_model, mode):
    pmeta, ids = fixture_ids
    meta, z = _golden()
    names = [pmeta["classnames"][c] for c in meta["classes"]]
    tok = _FixtureTokenizer(pmeta, ids)
    clf = Z.build_zero_shot_classifier(golden_model, tok, names, pmeta["templates"], use_tqdm=False, precision=mode)
    ref_clf = z[f"classifier_{mode}"]
    gap = meta["gap_fp32_fp64"] if mode == "fp32" else meta["gap_bf16_fp64"]
    d_clf = float(np.abs(clf.cpu().numpy() - ref_clf).max())
    print(f"{mode}: classifier max |diff| {d_clf:.3e} = {d_clf / gap['classifier']:.2f} x the golden's "
          f"{'fp32' if mode == 'fp32' else 'bf16'}-vs-fp64 gap")
    # measured on an H100: 29.7x the fp32-vs-fp64 gap in fp32 mode (2.1e-6 on unit-norm rows: the CPU run's rounding
    # errors mostly cancel in the 80-template mean, the device's bf16x3 text tower's do not), see the bf16 line below
    assert d_clf <= (64 if mode == "fp32" else 4) * gap["classifier"]
    x = seeded_images(meta["n_images"], meta["image_size"], meta["image_size"], seed=meta["image_seed"]).cuda()
    targets = torch.from_numpy(z["targets"]).cuda()
    ev = Z.ZeroShotEvaluator(golden_model, clf, precision=mode)
    for s in range(0, len(x), 32):
        ev.add(x[s:s + 32], targets[s:s + 32])
    ranks = ev.ranks().cpu().numpy()
    ref_logits, ref_ranks = z[f"logits_{mode}"].astype(np.float64), z[f"ranks_{mode}"]
    tgt = z["targets"]
    lt = ref_logits[np.arange(len(tgt)), tgt]
    bound = 2 * gap["logits"]
    near = (np.abs(ref_logits - lt[:, None]) <= bound).sum(1) > 1      # another class within the bound
    ambiguous = near.copy()
    if mode == "bf16":
        for i in range(len(tgt)):
            srt = np.sort(ref_logits[i])[::-1]
            ambiguous[i] |= any(srt[k - 1] == srt[k] and lt[i] == srt[k] for k in (1, 5))
    mism = (ranks != ref_ranks) & ~ambiguous
    print(f"{mode}: {int(ambiguous.sum())} ambiguous rows, {int((ranks != ref_ranks).sum())} rank differences")
    assert not mism.any(), np.nonzero(mism)
    top1, top5 = ev.result()
    n = len(tgt)
    c = meta["counts"][mode]
    assert abs(top1 - c["top1"]) * n / 100 <= ambiguous.sum() + 1e-9
    assert abs(top5 - c["top5"]) * n / 100 <= ambiguous.sum() + 1e-9
    ev.close()


# ------------------------------------------------------------------------------------------------ evaluator behaviour
@pytest.fixture(scope="module")
def small_setup():
    m = _model(preset("tiny", image_size=64))
    g = torch.Generator().manual_seed(11)
    clf = torch.nn.functional.normalize(torch.randn(128, 37, generator=g), dim=0).cuda()
    x = seeded_images(100, 64, 64, seed=12).cuda()
    t = torch.randint(0, 37, (100,), generator=g).cuda()
    return m, clf, x, t


def _run_batches(m, clf, x, t, mode, use_graph, bs=24, dtype=torch.float32):
    ev = Z.ZeroShotEvaluator(m, clf, precision=mode, use_graph=use_graph)
    for s in range(0, len(x), bs):                      # 100 = 4 x 24 + 4: a ragged last batch
        ev.add(x[s:s + bs].to(dtype), t[s:s + bs])
    r = ev.ranks().cpu()
    res = ev.result()
    ev.close()
    return r, res


@pytest.mark.parametrize("mode", ["fp32", "bf16"])
def test_graph_replay_equals_eager(small_setup, mode):
    m, clf, x, t = small_setup
    r0, res0 = _run_batches(m, clf, x, t, mode, False)
    r1, res1 = _run_batches(m, clf, x, t, mode, True)
    assert torch.equal(r0, r1) and res0 == res1


def test_bf16_images_equal_fp32_images_in_bf16_mode(small_setup):
    m, clf, x, t = small_setup
    r0, res0 = _run_batches(m, clf, x, t, "bf16", True)
    r1, res1 = _run_batches(m, clf, x, t, "bf16", True, dtype=torch.bfloat16)
    assert torch.equal(r0, r1) and res0 == res1


def test_add_does_not_synchronise_and_result_is_the_reference_formula(small_setup):
    m, clf, x, t = small_setup
    ev = Z.ZeroShotEvaluator(m, clf, precision="bf16")
    ev.add(x[:24], t[:24])                              # eager batch (first use of the shape)
    ev.add(x[24:48], t[24:48])                          # capture (synchronises once per shape)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        ev.add(x[:24], t[:24])                          # graph replays and a new shape's eager batch
        ev.add(x[48:72], t[48:72])
        ev.add(x[72:100], t[72:100])
    finally:
        torch.cuda.set_sync_debug_mode(0)
    ranks = ev.ranks().cpu().numpy()
    assert ev.result() == tuple(Z.accuracy_from_ranks(ranks, (1, 5)))
    ev.close()


# ------------------------------------------------------------------------------------------------ CLI
def _image_folder(root, classes, per_class, size, seed):
    from PIL import Image

    g = np.random.default_rng(seed)
    for ci, c in enumerate(classes):
        os.makedirs(os.path.join(root, c), exist_ok=True)
        for j in range(per_class):
            arr = g.integers(0, 256, (size + 3 * j, size + 5 * ci, 3), dtype=np.uint8)
            ext = "png" if (ci + j) % 2 else "jpg"
            Image.fromarray(arr).save(os.path.join(root, c, f"{j}.{ext}"))


def test_cli_end_to_end(tmp_path, capsys):
    from torch.utils.data import DataLoader
    from torchvision.datasets import ImageFolder

    from vtp_b200.text_tokenizer import BPETokenizer

    bpe = os.path.join(GOLDEN, "bpe_prefix.txt.gz")
    vocab = BPETokenizer(bpe_path=bpe).vocab_size
    m = _model(preset("tiny", image_size=64, text_vocab_size=vocab))
    ckpt = str(tmp_path / "ckpt")
    m.save_pretrained(ckpt)
    classes = ["bird", "car", "dog"]
    data = str(tmp_path / "data")
    _image_folder(data, classes, 7, 48, seed=5)
    prompts = tmp_path / "prompts.json"
    names, templates = ["a small bird", "a red car", "a dog"], ["a photo of a {c}.", "a drawing of the {c}.", "{c}"]
    prompts.write_text(json.dumps({"classnames": names, "templates": templates}))
    args = ["--model_path", ckpt, "--data_path", data, "--batch_size", "8", "--num_workers", "0", "--prompts",
            str(prompts), "--bpe_path", bpe]
    for prec in ("fp32", "bf16"):
        res = Z.main(args + ["--precision", prec])
        out = capsys.readouterr().out
        top1 = float(re.search(r"Top-1 Accuracy: ([0-9.]+)%", out).group(1))
        top5 = float(re.search(r"Top-5 Accuracy: ([0-9.]+)%", out).group(1))
        tok = BPETokenizer(bpe_path=bpe, context_length=77)
        loader = DataLoader(ImageFolder(data, transform=Z.make_transform(64)), batch_size=8, num_workers=0)
        clf = Z.build_zero_shot_classifier(m, tok, names, templates, use_tqdm=False, precision=prec)
        api = Z.evaluate(m, clf, loader, torch.device("cuda"), prec)
        assert (res["top1"], res["top5"]) == api
        assert (top1, top5) == (round(api[0], 2), round(api[1], 2))
        assert api[1] == 100.0                            # 3 classes: every target is in the top 5
    prompts.write_text(json.dumps({"classnames": names[:2], "templates": templates}))
    with pytest.raises(ValueError, match="3 classes"):
        Z.main(args)
