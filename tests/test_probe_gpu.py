"""Linear probe kernels and the device probe (vtp_b200/probe.py, csrc/probe.cu) against torch."""
import json
import os

import numpy as np
import pytest
import torch

from oracle.probe_taps import linear_input, probe_taps
from oracle.seeded import seeded_images, seeded_state_dict
from tests.util import load_golden
from vtp_b200 import lib
from vtp_b200 import probe as P
from vtp_b200.config import preset
from vtp_b200.model import VTPModel

pytestmark = pytest.mark.gpu


def _model(norm="rmsnorm", depth=4, seed=0):
    cfg = preset("tiny", vision_depth=depth, vision_norm_layer=norm)
    m = VTPModel(cfg)
    m.load_state_dict(seeded_state_dict({k: list(v.shape) for k, v in m.state_dict().items()}, seed=seed))
    return m.cuda()


def _reference_features(m, x, nmax, mode):
    """create_linear_input(n = nmax) over get_intermediate_layers_feature (linear_probing_hf.py:125-152)."""
    with torch.autocast("cuda", dtype=torch.bfloat16, enabled=(mode == "bf16")):
        feats = m.get_intermediate_layers_feature(x, n=nmax, return_class_token=True)
    return torch.cat([c for _, c in feats] + [feats[-1][0].mean(dim=1)], dim=-1).float()


@pytest.mark.parametrize("norm", ["rmsnorm", "layernorm"])
@pytest.mark.parametrize("mode", ["bf16", "fp32"])
@pytest.mark.parametrize("hw", [(224, 224), (256, 256), (160, 224)])
def test_features_match_intermediate_layers(norm, mode, hw):
    m = _model(norm)
    probe = P.LinearProbe(m, 37, batch_size=4, max_iter=4, precision=mode)
    x = seeded_images(4, *hw, seed=1).cuda()
    X = probe.features(x)
    ref = _reference_features(m, x, 4, mode)
    D = m.config.vision_embed_dim
    assert X.shape == ref.shape == (4, 5 * D)
    # the cls columns repeat vtp_norm_fwd's arithmetic; the patch mean differs from torch.mean in summation order only
    scale = ref[:, :4 * D].abs().mean().item()
    e_cls = (X[:, :4 * D] - ref[:, :4 * D]).abs().max().item() / scale
    e_mean = (X[:, 4 * D:] - ref[:, 4 * D:]).abs().max().item() / scale
    print(f"features {norm} {mode} {hw}: cls {e_cls:.2e}, patch mean {e_mean:.2e}")
    assert e_cls == 0.0 and e_mean < 1e-5, (e_cls, e_mean)


@pytest.mark.parametrize("C", [37, 1000])
def test_cross_entropy_matches_fp64(C):
    B, G = 64, 3
    Cp = (C + 7) // 8 * 8
    gen = torch.Generator().manual_seed(C)
    Z = (torch.randn(B, G * Cp, generator=gen) * 4).cuda()
    Z.view(B, G, Cp)[:5, :, :C] *= 20                        # rows with logits up to ±80
    Z.view(B, G, Cp)[5, :, 0] = 80.0
    Z.view(B, G, Cp)[6, :, C - 1] = -80.0
    labels = torch.randint(0, C, (B,), generator=gen)
    labels[:3] = torch.tensor([0, C - 1, 0])
    labels[5], labels[6] = 0, C - 1
    labels = labels.cuda()
    loss = torch.zeros(G, device="cuda")
    dZ3 = torch.full((3 * B, G * Cp), 7.0, dtype=torch.bfloat16, device="cuda")
    db = torch.full((G * Cp,), 7.0, device="cuda")
    lib.probe_ce(Z, B, G, C, Cp, labels, loss, dZ3, db)
    dZ = dZ3[:B].double() + dZ3[2 * B:].double()
    assert torch.equal(dZ3[:B], dZ3[B:2 * B])
    for g in range(G):
        z = Z.view(B, G, Cp)[:, g, :C].double().requires_grad_(True)
        ref = torch.nn.functional.cross_entropy(z, labels)
        ref.backward()
        assert abs(loss[g].item() - ref.item()) <= 1e-5 * max(1.0, ref.item())
        got = dZ.view(B, G, Cp)[:, g]
        # hi + lo carries dZ to 2^-17 relative; fp32 softmax adds a few ulp of the probability / B
        assert ((got[:, :C] - z.grad).abs() <= 2.0 ** -16 * z.grad.abs() + 1e-9).all()
        assert torch.all(got[:, C:] == 0)
        dbg = db.view(G, Cp)[g].double()
        assert (dbg[:C] - z.grad.sum(0)).abs().max().item() < 5e-7 and torch.all(dbg[C:] == 0)


def test_sgd_matches_torch_and_refreshes_operand():
    G, Cp, K, steps = 3, 8, 16, 20
    lrs = [0.05, 0.01, 0.002]
    tab = torch.from_numpy(P.lr_table(lrs, steps)).cuda()
    gen = torch.Generator().manual_seed(0)
    w0 = torch.randn(G, Cp, K, generator=gen).cuda()
    grads = [torch.randn(G, Cp, K, generator=gen).cuda() for _ in range(steps)]
    params = [torch.nn.Parameter(w0[i].clone()) for i in range(G)]
    opt = torch.optim.SGD([{"params": [p], "lr": lr} for p, lr in zip(params, lrs)], momentum=0.9, weight_decay=0)
    sched = torch.optim.lr_scheduler.CosineAnnealingLR(opt, steps, eta_min=0)
    p, buf = w0.clone().reshape(-1), torch.zeros(G * Cp * K, device="cuda")
    pb = torch.empty(G * Cp, 3 * K, dtype=torch.bfloat16, device="cuda")
    hyper = torch.zeros(8, device="cuda")
    max_ulp = 0
    for t in range(steps):
        for i, prm in enumerate(params):
            prm.grad = grads[t][i].clone()
        opt.step()
        sched.step()
        lib.hyper_tick(hyper, 0.0, 0.0)
        lib.probe_sgd(p, grads[t].reshape(-1), buf, p.numel(), row_len=K, rows_per_cls=Cp, cls0=0, lr_table=tab,
                      hyper=hyper, momentum=0.9, pb=pb)
        want = torch.stack([prm.detach() for prm in params]).reshape(-1)
        ulp = (p.view(torch.int32).long() - want.view(torch.int32).long()).abs().max().item()
        max_ulp = max(max_ulp, ulp)
    print(f"SGD: {max_ulp} ulp from torch.optim.SGD over {steps} steps")
    assert max_ulp == 0, f"{max_ulp} ulp from torch.optim.SGD"
    ref_pb = torch.empty_like(pb)
    lib.split3(p.view(G * Cp, K), ref_pb, G * Cp, K, b_side=True)
    assert torch.equal(pb, ref_pb)


def test_top1_counts_follow_torch_argmax():
    B, G, C = 200, 4, 37
    Cp = 40
    gen = torch.Generator().manual_seed(1)
    Z = torch.randint(-3, 4, (B, G * Cp), generator=gen).float()       # many ties
    Z.view(B, G, Cp)[:, :, C:] = 1e9                                   # padding never wins
    Z.view(B, G, Cp)[10:20, 1, 5] = float("nan")
    Z.view(B, G, Cp)[15:20, 1, 2] = float("nan")
    Z.view(B, G, Cp)[30, 2, :C] = float("nan")
    Z.view(B, G, Cp)[31, 3, :C] = float("-inf")
    labels = torch.randint(0, C, (B,), generator=gen)
    labels[10:20] = 5
    labels[15:17] = 2
    Zc, lc = Z.cuda(), labels.cuda()
    counts = torch.zeros(G, dtype=torch.int64, device="cuda")
    lib.probe_correct(Zc, B, G, C, Cp, lc, counts)
    lib.probe_correct(Zc, B, G, C, Cp, lc, counts)
    want = torch.stack([(Z.view(B, G, Cp)[:, g, :C].argmax(1) == labels).sum() for g in range(G)])
    assert torch.equal(counts.cpu(), 2 * want)


def test_classifier_step_matches_fp64_sgd_step():
    m = _model()
    B, C = 32, 37
    probe = P.LinearProbe(m, C, batch_size=B, max_iter=10)
    gen = torch.Generator().manual_seed(2)
    X = torch.randn(B, probe.KX, generator=gen).cuda()
    labels = torch.randint(0, C, (B,), generator=gen).cuda()
    before = probe.state_dict()
    probe.classifier_step(X, labels)
    after = probe.state_dict()
    losses = probe.take_losses().cpu()
    Xd, D = X.double().cpu(), probe.D
    for i, c in enumerate(probe.classifiers):
        k = f"classifiers_dict.{c.key}.linear."
        w = before[k + "weight"].double().requires_grad_(True)
        b = before[k + "bias"].double().requires_grad_(True)
        x = Xd[:, (probe.nmax - c.n) * D:]
        loss = torch.nn.functional.cross_entropy(x @ w.T + b, labels.cpu())
        loss.backward()
        assert abs(losses[i].item() - loss.item()) < 1e-5 * loss.item()
        lr = float(np.float32(c.lr))
        for name, prm in (("weight", w), ("bias", b)):
            step = after[k + name].double() - before[k + name].double()
            ref = -lr * prm.grad
            # the fp32 parameter rounds the step to its own ulp
            tol = 1e-4 * ref.abs().max().item() + 2.0 ** -23 * before[k + name].double().abs() + 1e-12
            assert ((step - ref).abs() <= tol).all(), (c.key, name)


def test_classifier_step_rejects_unchecked_inputs():
    probe = P.LinearProbe(_model(), 37, batch_size=8, max_iter=2)
    X = torch.randn(8, probe.KX + 8, device="cuda")
    y = torch.zeros(8, dtype=torch.int64, device="cuda")
    with pytest.raises(ValueError):
        probe.classifier_step(X[:, 8:], y)                      # strided view
    with pytest.raises(ValueError):
        probe.classifier_step(X[:, 8:].contiguous(), y.int())   # int32 labels


# bf16x3 products carry 16 significant bits where fp32 carries 24: its rounding is 2^8 times fp32's
BF16X3_OVER_FP32 = 2.0 ** 8


def test_golden_run_matches_reference():
    """tests/golden/probe_tiny.* is the reference's own setup_linear_classifiers / train_one_epoch / evaluate on seeded
    taps (oracle/make_golden_probe.py).  Tolerances: the stored fp32-vs-fp64 gap of the reference run, times 2^8."""
    meta, g = load_golden("probe_tiny")
    C, B, steps = meta["C"], meta["B"], meta["steps"]
    cfg = preset("tiny", vision_embed_dim=meta["D"], vision_num_heads=1, vision_depth=4, train_clip=False,
                 train_reconstruction=False)
    probe = P.LinearProbe(VTPModel(cfg).cuda(), C, batch_size=B, max_iter=steps, seed=meta["seed"], use_graph=False)
    assert probe.keys == meta["keys"] and probe.G == 24
    F = BF16X3_OVER_FP32
    losses = []
    for t in range(steps):
        feats, labels = probe_taps(t)
        probe.classifier_step(linear_input(feats, 4).float().contiguous().cuda(), labels.cuda())
        losses.append(probe.take_losses().cpu())
    e = (torch.stack(losses).double() - g["loss"].double()).abs().max().item()
    print(f"golden: loss {e:.2e} (gap {g['gap_loss'].max().item():.2e})")
    assert e <= F * g["gap_loss"].max().item()
    sd = probe.state_dict()
    tw = F * g["gap_weight"].max().item()
    worst = 0.0
    for i, k in enumerate(meta["keys"]):
        w = sd[f"classifiers_dict.{k}.linear.weight"].double()
        b = sd[f"classifiers_dict.{k}.linear.bias"].double()
        worst = max(worst, (w[meta["weight_rows"]] - g[f"w{i}"].double()).abs().max().item())
        assert (w[meta["weight_rows"]] - g[f"w{i}"].double()).abs().max().item() <= tw, k
        assert (w.norm(dim=1) - g["row_norm"][i]).abs().max().item() <= tw * w.shape[1] ** 0.5, k
        assert (b - g["bias"][i].double()).abs().max().item() <= F * g["gap_bias"].max().item(), k
    print(f"golden: weights {worst:.2e} (gap {g['gap_weight'].max().item():.2e})")
    feats, labels = probe_taps(-1, meta["n_eval"])
    Z = probe.logits(linear_input(feats, 4).float().contiguous().cuda())
    counts = torch.zeros(probe.G, dtype=torch.int64, device="cuda")
    lib.probe_correct(Z, Z.shape[0], probe.G, C, probe.Cp, labels.cuda(), counts)
    ours = (Z.view(-1, probe.G, probe.Cp)[:, :, :C].argmax(-1).cpu() == labels[:, None]).T   # [G, n_eval]
    sure = g["margin"].double() > F * g["gap_margin"].item()
    assert torch.equal(ours[sure], g["correct"][sure])
    n = meta["n_eval"]
    for i in range(probe.G):
        ref = round(g["acc"][i].item() * n / 100)
        assert int(counts[i]) == int(ours[i].sum())
        assert abs(int(counts[i]) - ref) <= int((~sure[i]).sum()), meta["keys"][i]
    print(f"golden: {int((~sure).sum())} low-margin (row, classifier) pairs of {sure.numel()}")


def test_graph_replay_is_bit_identical_to_eager():
    m = _model()
    B, C = 8, 37
    probes = [P.LinearProbe(m, C, batch_size=B, max_iter=8, use_graph=g) for g in (False, True)]
    for t in range(4):
        x = seeded_images(B, 64, 64, seed=10 + t).cuda()
        y = torch.arange(B, device="cuda") * 3 % C
        for pr in probes:
            pr.train_step(x, y)
    assert probes[0]._graph.graph is None and probes[1]._graph.graph is not None
    a, b = probes
    assert torch.equal(a.p, b.p) and torch.equal(a.buf, b.buf) and torch.equal(a.loss_acc, b.loss_acc)
    assert torch.equal(a.wb[0], b.wb[0]) and torch.equal(a.wb[1], b.wb[1])
    probes[1].release()


def _image_folder(root, n_per_class, seed):
    from PIL import Image

    rng = np.random.default_rng(seed)
    colours = [(200, 40, 40), (40, 200, 40), (40, 40, 200)]
    for split, n in (("train", n_per_class), ("val", n_per_class // 2)):
        for ci, col in enumerate(colours):
            d = os.path.join(root, split, f"class{ci}")
            os.makedirs(d, exist_ok=True)
            for i in range(n):
                img = np.clip(np.asarray(col)[None, None] + rng.normal(0, 30, (48, 64, 3)), 0, 255).astype(np.uint8)
                Image.fromarray(img).save(os.path.join(d, f"{i}.png"))


def test_cli_end_to_end(tmp_path):
    _image_folder(str(tmp_path / "data"), 32, seed=0)
    m = _model()
    m.save_pretrained(str(tmp_path / "ckpt"))
    out = tmp_path / "out"
    res = P.main(["--model_path", str(tmp_path / "ckpt"), "--imagenet_root", str(tmp_path / "data"), "--output_dir", str(out),
                  "--batch_size", "32", "--epochs", "2", "--epoch_length", "12", "--num_workers", "0"])
    with open(out / "linear_probing_results.json") as f:
        saved = json.load(f)
    assert set(saved) == {"best_accuracy", "best_classifier", "all_accuracies"}
    keys = [c.key for c in P.plan_classifiers((1, 4), P.DEFAULT_LEARNING_RATES, 32)[0]]
    assert list(saved["all_accuracies"]) == keys and saved["best_classifier"] in keys
    assert saved["best_accuracy"] == res["best_accuracy"] > 100.0 / 3 + 20


def _free_port():
    import socket

    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _dist_worker(rank, world, port, out):
    import torch.distributed as dist

    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    m = _model()
    Bg, C = 16, 37
    B = Bg // world
    mine = slice(rank * B, (rank + 1) * B)
    sharded = P.LinearProbe(m, C, batch_size=B, max_iter=6)            # world 2 from torch.distributed
    single = P.LinearProbe(m, C, batch_size=Bg, max_iter=6, world=1)   # the global batch in one process
    assert sharded.world == world and sharded.keys == single.keys
    val = [(seeded_images(Bg, 64, 64, seed=40 + i), torch.arange(Bg) * 7 % C) for i in range(2)]
    acc_sharded = sharded.evaluate([(x[mine], y[mine]) for x, y in val])
    acc_single = single.evaluate(val)
    for t in range(4):                    # step 1 eager, then the captured graph with the all-reduce inside
        x = seeded_images(Bg, 64, 64, seed=10 + t).cuda()
        y = (torch.arange(Bg, device="cuda") * 5 + t) % C
        sharded.train_step(x[mine], y[mine])
        single.train_step(x, y)
    sharded.release()
    single.release()
    rel = ((sharded.p - single.p).norm() / single.p.norm()).item()
    other = sharded.p.clone()
    dist.broadcast(other, src=0)
    out[rank] = (acc_sharded == acc_single, rel, torch.equal(other, sharded.p))
    dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_rank_probe_equals_global_batch():
    """Each rank takes half of the batch: the all-reduced counts equal the single-process counts, and after four steps
    (gradient all-reduce inside the step graph, averaged by grad_scale = 1/world) the classifiers equal the
    single-process run on the whole batch up to summation order, and stay identical across ranks."""
    import torch.multiprocessing as mp

    world, port = 2, _free_port()
    mgr = mp.Manager()
    out = mgr.dict()
    mp.spawn(_dist_worker, args=(world, port, out), nprocs=world, join=True)
    for r in range(world):
        same_acc, rel, same_across = out[r]
        assert same_acc
        assert rel < 1e-6, rel
        assert same_across
