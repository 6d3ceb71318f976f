"""FID host side (vtp_b200/fid.py) and the reference network (oracle/fid_inception.py), without a GPU: the weight loader
and BatchNorm folding, the FID blocks against torchvision's, the Fréchet distance, the file listing, the statistics file
and mu / sigma from the accumulated sums."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle.fid_inception import FIDInceptionA, FIDInceptionC, FIDInceptionE_1, FIDInceptionE_2, fid_inception
from vtp_b200 import fid


def _torchvision_state(seed=0):
    """A torchvision-layout Inception3 state dict with random values (fc of 1008 classes, num_batches_tracked)."""
    torch.manual_seed(seed)
    net = fid_inception(None, dtype=torch.float32)
    sd = {k: (torch.randn_like(v) if v.is_floating_point() else v) for k, v in net.state_dict().items()}
    for k in sd:
        if k.endswith("running_var"):
            sd[k] = sd[k].abs() + 0.1
    assert sd["fc.weight"].shape == (1008, 2048)
    return sd


def test_loader_accepts_torchvision_layout_and_names_missing_keys(tmp_path):
    sd = _torchvision_state()
    torch.save(sd, tmp_path / "w.pth")
    got = fid.load_weight_file(str(tmp_path / "w.pth"))
    assert sorted(got) == sorted(fid.required_keys()) and len(got) == 94 * 5
    assert not any(k.startswith(("fc.", "AuxLogits.")) or "num_batches" in k for k in got)
    del sd["Mixed_6c.branch7x7dbl_4.bn.running_var"]
    torch.save(sd, tmp_path / "bad.pth")
    with pytest.raises(KeyError, match="Mixed_6c.branch7x7dbl_4.bn.running_var"):
        fid.load_weight_file(str(tmp_path / "bad.pth"))


@pytest.mark.parametrize("name", ["Conv2d_1a_3x3", "Mixed_5b.branch5x5_2", "Mixed_6e.branch7x7dbl_5", "Mixed_7c.branch3x3_2b"])
def test_bn_folding_equals_conv_bn_in_fp64(name):
    sd = _torchvision_state(1)
    net = fid_inception(sd, dtype=torch.float64)
    mod = net
    for part in name.split("."):
        mod = getattr(mod, part)
    ci = fid.CONVS[name][0]
    x = torch.randn(2, ci, 11, 13, dtype=torch.float64)
    with torch.no_grad():
        want = mod.bn(mod.conv(x))                                  # conv + eval BN in fp64, before the ReLU
    w, b = fid.fold_bn(sd, name)
    # the fold is done in fp64 and rounded once to fp32
    s = sd[f"{name}.bn.weight"].double() / torch.sqrt(sd[f"{name}.bn.running_var"].double() + 1e-3)
    assert torch.equal(w, (sd[f"{name}.conv.weight"].double() * s[:, None, None, None]).float())
    got = F.conv2d(x, w.double(), b.double(), mod.conv.stride, mod.conv.padding)
    mag = F.conv2d(x.abs(), w.double().abs(), b.double().abs(), mod.conv.stride, mod.conv.padding)
    assert ((got - want).abs() <= 2.0 ** -23 * mag + 1e-12).all()


def _copy_weights(dst, src):
    dst = dst.double()
    dst.load_state_dict(src.state_dict())
    return dst.eval()


def test_fid_blocks_differ_from_torchvision_exactly_at_the_pool():
    from torchvision.models.inception import InceptionA, InceptionC, InceptionE

    torch.manual_seed(0)
    cases = [(InceptionA(8, pool_features=8), FIDInceptionA, dict(pool_features=8)),
             (InceptionC(8, channels_7x7=8), FIDInceptionC, dict(channels_7x7=8)),
             (InceptionE(8), FIDInceptionE_1, {})]
    x = torch.rand(2, 8, 7, 9, dtype=torch.float64) + 0.5
    for tv, cls, kw in cases:
        tv = tv.double().eval()
        for m in tv.modules():
            if isinstance(m, torch.nn.BatchNorm2d):
                m.running_mean.uniform_(-0.1, 0.1)
                m.running_var.uniform_(0.5, 2.0)
        ours = _copy_weights(cls(8, **kw), tv)
        with torch.no_grad():
            a, b = tv(x), ours(x)
        # every branch but the pool branch is the same; the pool branch's 1x1 conv sees count_include_pad=False
        # averages, which equal torchvision's only on interior pixels
        C = a.shape[1]
        pool_c = {FIDInceptionA: 8, FIDInceptionC: 192, FIDInceptionE_1: 192}[cls]
        assert torch.equal(a[:, :C - pool_c], b[:, :C - pool_c])
        assert torch.allclose(a[:, C - pool_c:, 1:-1, 1:-1], b[:, C - pool_c:, 1:-1, 1:-1], rtol=1e-12, atol=1e-12)
        border = torch.ones(7, 9, dtype=torch.bool)
        border[1:-1, 1:-1] = False
        assert (a[:, C - pool_c:][..., border] - b[:, C - pool_c:][..., border]).abs().max() > 1e-3
    tv = InceptionE(8).double().eval()
    e2 = _copy_weights(FIDInceptionE_2(8), tv)
    e1 = _copy_weights(FIDInceptionE_1(8), tv)
    with torch.no_grad():
        a, b, c = tv(x), e2(x), e1(x)
    assert torch.equal(a[:, :-192], b[:, :-192])
    assert (a[:, -192:, 1:-1, 1:-1] - b[:, -192:, 1:-1, 1:-1]).abs().max() > 1e-3     # max pool, not average
    with torch.no_grad():
        mp = F.max_pool2d(x, 3, 1, 1)
        assert torch.allclose(b[:, -192:], e2.branch_pool(mp), rtol=0, atol=0)
    assert torch.allclose(a[:, -192:, 1:-1, 1:-1], c[:, -192:, 1:-1, 1:-1], rtol=1e-12, atol=1e-12)


# ---------------------------------------------------------------------------------------------------------- distance
def test_frechet_diagonal_closed_form():
    rng = np.random.default_rng(0)
    mu1, mu2 = rng.normal(size=16), rng.normal(size=16)
    a, b = rng.uniform(0.1, 3, 16), rng.uniform(0.1, 3, 16)
    want = np.sum((mu1 - mu2) ** 2) + np.sum((np.sqrt(a) - np.sqrt(b)) ** 2)
    assert fid.frechet_distance(mu1, np.diag(a), mu2, np.diag(b)) == pytest.approx(want, rel=1e-12)


def test_frechet_identical_statistics_is_zero():
    rng = np.random.default_rng(1)
    x = rng.normal(size=(200, 32))
    mu, s = x.mean(0), np.cov(x, rowvar=False)
    assert abs(fid.frechet_distance(mu, s, mu, s)) <= 1e-10 * np.trace(s)


def test_frechet_singular_product_takes_eps_path(capsys):
    rng = np.random.default_rng(2)
    mu1, mu2 = rng.normal(size=3), rng.normal(size=3)
    s1 = np.zeros((3, 3))
    b = rng.uniform(0.5, 2, 3)
    got = fid.frechet_distance(mu1, s1, mu2, np.diag(b))
    assert "singular product" in capsys.readouterr().out
    eps = 1e-6
    want = np.sum((mu1 - mu2) ** 2) + np.sum(b) - 2 * np.sum(np.sqrt(eps * (b + eps)))
    assert got == pytest.approx(want, rel=1e-9)


def test_frechet_large_imaginary_part_raises():
    with pytest.raises(ValueError, match="Imaginary component"):
        fid.frechet_distance(np.zeros(2), np.eye(2), np.zeros(2), np.diag([1.0, -1.0]))


# ---------------------------------------------------------------------------------------------------------- files
def test_directory_listing_rules(tmp_path):
    names = ["b.png", "a.jpg", "c.JPG", "d.webp", "e.txt", "f.jpeg", "g.tiff", "h.PNG", "i.bmp", "j.pgm", "k.ppm",
             "l.tif", "m.gif"]
    for n in names:
        (tmp_path / n).write_bytes(b"")
    (tmp_path / "sub").mkdir()
    (tmp_path / "sub" / "x.png").write_bytes(b"")
    got = [p.name for p in fid.list_images(str(tmp_path))]
    assert got == sorted(["b.png", "a.jpg", "d.webp", "f.jpeg", "g.tiff", "i.bmp", "j.pgm", "k.ppm", "l.tif"])


def test_npz_round_trip_keeps_pytorch_fid_keys_and_dtypes(tmp_path):
    rng = np.random.default_rng(3)
    mu, sigma = rng.normal(size=8), np.cov(rng.normal(size=(20, 8)), rowvar=False)
    p = str(tmp_path / "s.npz")
    fid.save_stats_npz(p, mu, sigma)
    with np.load(p) as f:
        assert sorted(f.files) == ["mu", "sigma"]
        assert f["mu"].dtype == np.float32 and f["sigma"].dtype == np.float64
    m2, s2 = fid.statistics_of_path(p, model=None)
    assert np.array_equal(m2, mu.astype(np.float32)) and np.array_equal(s2, sigma)


def test_invalid_path_and_dims():
    with pytest.raises(RuntimeError, match="Invalid path"):
        fid.fid_from_paths(["/nonexistent/a", "/nonexistent/b"], weights="w")
    with pytest.raises(NotImplementedError):
        fid.fid_from_paths(["a", "b"], dims=768)


def test_mu_sigma_from_sums_equals_numpy():
    rng = np.random.default_rng(4)
    D, n = 128, 300
    x = rng.normal(size=(n, D)) * rng.uniform(0.1, 2, D) + rng.uniform(0, 1, D)
    st = fid.FIDStatistics(device="cpu", dims=D)
    st.S2.copy_(torch.from_numpy(np.triu(x.T @ x)))          # the device fills the upper triangle only
    st.S1.copy_(torch.from_numpy(x.sum(0)))
    st.n.fill_(n)
    mu, sigma = st.mu_sigma()
    want_s = np.cov(x, rowvar=False)
    assert np.abs(mu - np.mean(x, 0)).max() <= 1e-12 * np.abs(x).max()
    assert np.linalg.norm(sigma - want_s) <= 1e-12 * np.linalg.norm(want_s)
    assert np.array_equal(sigma, sigma.T)
