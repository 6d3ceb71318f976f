"""Host side of the linear probe (vtp_b200/probe.py): classifier keys, the lr table, the CLI flags."""
import numpy as np
import pytest
import torch

from vtp_b200 import probe as P


def _reference_module_dict_keys(ns, lrs, batch_size, world):
    """Restates linear_probing_hf.py:233-246 with torch's own ModuleDict: which keys survive, in which order, and which
    created classifier each key ends up holding."""
    d = torch.nn.ModuleDict()
    created = 0
    for n in ns:
        for lr in lrs:
            s = P.scale_lr(lr, batch_size, world)
            m = torch.nn.Identity()
            m.created = created
            created += 1
            d[P.classifier_key(n, s)] = m
    return [(k, m.created) for k, m in d.items()], created


@pytest.mark.parametrize("world,expect", [(1, 24), (8, 26)])
def test_classifier_keys_follow_module_dict(world, expect):
    plan, created = P.plan_classifiers((1, 4), P.DEFAULT_LEARNING_RATES, 128, world)
    ref, ref_created = _reference_module_dict_keys((1, 4), P.DEFAULT_LEARNING_RATES, 128, world)
    assert created == ref_created == 26
    assert len(plan) == expect
    assert [(c.key, c.created) for c in plan] == ref
    for c in plan:
        assert c.key == P.classifier_key(c.n, c.lr)


def test_keys_equal_the_reference_run():
    """tests/golden/probe_tiny.json holds the keys of the reference's own setup_linear_classifiers (batch 128, world 1)."""
    import json
    import os

    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "probe_tiny.json")) as f:
        meta = json.load(f)
    plan, _ = P.plan_classifiers((1, 4), tuple(meta["lrs"]), meta["B"], 1)
    assert [c.key for c in plan] == meta["keys"] and len(plan) == 24


def test_colliding_keys_at_world_one():
    plan, _ = P.plan_classifiers((1, 4), P.DEFAULT_LEARNING_RATES, 128, 1)
    keys = [c.key for c in plan]
    assert keys[0] == "classifier_1_blocks_avgpool_True_lr_0_00001"
    assert keys[12] == "classifier_4_blocks_avgpool_True_lr_0_00001"
    # the key keeps the first classifier's place and holds the second one (lr 2e-5 * 128 / 256)
    assert plan[0].created == 1 and plan[0].lr == pytest.approx(1e-5, rel=0, abs=1e-20)
    assert plan[12].created == 14
    assert [c.n for c in plan] == [1] * 12 + [4] * 12


def test_lr_table_equals_torch_scheduler():
    lrs = [P.scale_lr(lr, 128) for lr in P.DEFAULT_LEARNING_RATES]
    max_iter = 57
    tab = P.lr_table(lrs, max_iter)
    assert tab.dtype == np.float32 and tab.shape == (max_iter, len(lrs))
    params = [torch.nn.Parameter(torch.randn(3)) for _ in lrs]
    opt = torch.optim.SGD([{"params": [p], "lr": lr} for p, lr in zip(params, lrs)], momentum=0.9, weight_decay=0)
    sched = torch.optim.lr_scheduler.CosineAnnealingLR(opt, max_iter, eta_min=0)
    for t in range(max_iter):
        want = np.asarray([g["lr"] for g in opt.param_groups], dtype=np.float64).astype(np.float32)
        assert np.array_equal(tab[t], want), t
        for p in params:
            p.grad = torch.ones_like(p)
        opt.step()
        sched.step()


def test_initial_weights_follow_reference_draw_order():
    ns, lrs, D, C = (1, 4), (1e-3, 1e-2), 8, 5
    got = P.initial_weights(ns, lrs, {n: (n + 1) * D for n in ns}, C, seed=3)
    torch.manual_seed(3)
    for i, n in enumerate(n for n in ns for _ in lrs):
        lin = torch.nn.Linear((n + 1) * D, C)
        lin.weight.data.normal_(mean=0.0, std=0.01)
        assert torch.equal(got[i][0], lin.weight.data) and torch.equal(got[i][1], torch.zeros(C))


def test_cli_parses_reference_flags():
    a = P.build_parser().parse_args([
        "--model_path", "m", "--imagenet_root", "r", "--output_dir", "o", "--batch_size", "64", "--epochs", "3",
        "--epoch_length", "7", "--num_workers", "2", "--device", "cuda:1", "--precision", "fp32", "--use_ddp",
        "--local_rank", "1"])
    assert (a.model_path, a.imagenet_root, a.output_dir, a.batch_size, a.epochs, a.epoch_length, a.num_workers, a.device,
            a.precision, a.use_ddp, a.local_rank) == ("m", "r", "o", 64, 3, 7, 2, "cuda:1", "fp32", True, 1)
    d = P.build_parser().parse_args(["--model_path", "m", "--imagenet_root", "r"])
    assert (d.batch_size, d.epochs, d.epoch_length, d.precision, d.use_ddp, d.output_dir) == \
        (128, 10, 1250, "bf16", False, "./linear_probing_results")
    with pytest.raises(SystemExit):
        P.build_parser().parse_args(["--model_path", "m"])


def test_transforms_are_the_reference_pipelines():
    tr, ev = P.make_transforms()
    names = [type(t).__name__ for t in tr.transforms]
    assert names == ["RandomResizedCrop", "RandomHorizontalFlip", "ToTensor", "Normalize"]
    assert [type(t).__name__ for t in ev.transforms] == ["Resize", "CenterCrop", "ToTensor", "Normalize"]
    assert tr.transforms[0].size == (224, 224) and ev.transforms[0].size == 256 and ev.transforms[1].size == (224, 224)
    assert str(tr.transforms[0].interpolation).endswith("BICUBIC") and str(ev.transforms[0].interpolation).endswith("BICUBIC")
