"""Saving and resuming a training run (VTPTrainer.save_checkpoint / load_checkpoint, TrainBatchPipeline.state_dict /
load_state_dict, export_state_dict(teacher=True)) on the tiny preset with LPIPS, cosine schedules and stochastic depth in
the self-distillation objective.

Everything a load restores is compared bit for bit.  Comparisons that cross a training step use the tolerances of
test_train_gpu.test_graph_step_equals_eager_steps: the split-K weight gradients accumulate with fp32 atomics, so two runs
of the same step are not bit-identical."""
import json
import os
import socket

import pytest
import torch

from oracle.seeded import seeded_captions, seeded_images
from tests.util import rel
from vtp_b200.config import preset
from vtp_b200.schedules import CosineSchedule
from vtp_b200.train import TrainConfig, VTPTrainer

pytestmark = pytest.mark.gpu

B, N_LOC, HW = 4, 2, 16


def _trainer(seed=0, K=512, device="cuda"):
    tc = TrainConfig(head_out_dim=K, head_hidden=256, head_bottleneck=64, n_local_crops=N_LOC, ssl_drop_rate=0.25)
    tr = VTPTrainer(preset("tiny"), tc, device=device)
    tr.reset_parameters(seed)
    tr.enable_lpips(seed=0, chunk=2)
    tr.set_schedules(lr=CosineSchedule(3e-4, 1e-5, total_iters=12, warmup_iters=2, start_warmup_value=1e-5),
                     teacher_momentum=CosineSchedule(0.99, 1.0, total_iters=12))
    return tr


def _batch(seed=0, device="cuda"):
    masks = torch.zeros(2 * B, HW, dtype=torch.bool)
    masks[::2, :5] = True
    return dict(image=seeded_images(B, 64, 64, seed=seed).to(device), text=seeded_captions(B, 77, 1000).to(device),
                global_crops=seeded_images(2 * B, 64, 64, seed=seed + 21).to(device),
                local_crops=seeded_images(N_LOC * B, 32, 32, seed=seed + 22).to(device),
                mask_indices=masks.flatten().nonzero().flatten().to(device),
                masks_weight=(1.0 / masks.sum(-1).clamp(min=1).float())[:, None].expand_as(masks)[masks].to(device),
                rec_image=seeded_images(B, 64, 64, seed=seed + 31).to(device))


def _state(tr):
    """Everything a load restores (and the bf16 copies it re-derives), cloned."""
    st = tr.store
    return dict(p=st.p.clone(), m=st.m.clone(), v=st.v.clone(), tp=st.tp.clone(), pb=st.pb.clone(), tpb=st.tpb.clone(),
                center_dino=tr.center_dino.clone(), center_ibot=tr.center_ibot.clone(), hyper=tr.hyper[0:3].clone(),
                step_count=tr.step_count)


def _assert_same(saved, tr):
    now = _state(tr)
    for k, v in saved.items():
        assert (v == now[k]) if k == "step_count" else torch.equal(v, now[k]), k


def _assert_track(la, lb, a, b):
    for x, y in zip(la, lb):
        assert torch.isfinite(y).all()
        assert torch.allclose(x, y, rtol=2e-3, atol=1e-5), (x, y)
    assert rel(b.store.p, a.store.p) < 1e-4
    assert rel(b.store.tp, a.store.tp) < 1e-5


def test_round_trip(tmp_path):
    batch = _batch()
    a = _trainer(0)
    for _ in range(3):
        a.train_step(batch)
    path = str(tmp_path / "ck")
    a.save_checkpoint(path)
    saved, rng = _state(a), torch.cuda.get_rng_state()
    assert saved["center_dino"].abs().max() > 0 and saved["m"].abs().max() > 0
    torch.rand(1000, device="cuda"), torch.randperm(7, device="cuda")        # A and B share this generator
    assert not torch.equal(torch.cuda.get_rng_state(), rng)
    b = _trainer(1)
    assert not torch.equal(b.store.p, a.store.p)
    assert b.load_checkpoint(path) == 3
    _assert_same(saved, b)                      # incl. pb / tpb: re-derived == what the fused AdamW kernel wrote
    assert torch.equal(torch.cuda.get_rng_state(), rng)
    # one more step of each, with the same stochastic-depth subsets: the lr comes from the table at the restored step
    la = a.train_step(batch).cpu().clone()
    torch.cuda.set_rng_state(rng)
    lb = b.train_step(batch).cpu().clone()
    _assert_track([la], [lb], a, b)
    assert a.scheduled_values() == b.scheduled_values()
    assert b.scheduled_values()["step"] == 4


def test_load_into_captured_graph(tmp_path):
    """The documented resume sequence: capture first (its warm-up steps train the fresh trainer), then load; the graph
    replays from the restored buffers, RNG state and step counter with no re-capture."""
    batch, b2 = _batch(0), _batch(5)
    seq = [batch, b2, batch]
    a = _trainer(0)
    for _ in range(3):
        a.train_step(batch)
    path = str(tmp_path / "ck")
    a.save_checkpoint(path)
    saved = _state(a)
    la = [a.train_step(x).cpu().clone() for x in seq]       # the uninterrupted run, from the saved RNG state
    b = _trainer(1)
    b.capture_step(batch, warmup=2)
    graph, launches = b._graph.graph, b.graph_launches
    b.load_checkpoint(path)
    _assert_same(saved, b)
    assert b._graph.graph is graph
    lb = [b.replay_step(x).cpu().clone() for x in seq]
    _assert_track(la, lb, a, b)
    assert b.scheduled_values() == a.scheduled_values()
    assert b.scheduled_values()["step"] == 3 + len(seq) and b.step_count == a.step_count
    c = _trainer(2)                                          # never loaded: the same graph
    c.capture_step(batch, warmup=1)
    assert c.graph_launches == launches


def _images(i):
    g = torch.Generator().manual_seed(100 + i)
    return torch.randint(0, 256, (B, 72, 88, 3), dtype=torch.uint8, generator=g).pin_memory()


def _pipe(seed):
    from vtp_b200.data import PhotometricAug, TrainBatchPipeline
    return TrainBatchPipeline("cuda", image_size=64, local_size=32, n_local=N_LOC, patch=16, seed=seed,
                              photometric=PhotometricAug())


def test_pipeline_resume(tmp_path):
    """Two batches in flight; the save after step s has batch s queued.  A new pipeline (another seed) loads the state,
    is given the images from batch s on, and prepares bit-identical batches; the resumed trainer tracks the
    uninterrupted one."""
    n, s = 6, 3
    ids = [seeded_captions(B, 77, 1000, seed=i) for i in range(n)]
    path = str(tmp_path / "ck")
    pa, a = _pipe(0), _trainer(0)
    pa.submit(_images(0), ids[0])
    got_a, la = [], []
    for i in range(n):
        if i + 1 < n:
            pa.submit(_images(i + 1), ids[i + 1])
        x = pa.get()
        got_a.append({k: v.clone() for k, v in x.items()})
        la.append(a.train_step(x).cpu().clone())
        if i + 1 == s:
            a.save_checkpoint(path, pipeline=pa)
    pa.close()
    pb, b = _pipe(5), _trainer(1)
    b.capture_step(got_a[0], warmup=1)
    with pytest.raises(ValueError, match="queued"):
        busy = _pipe(0)
        busy.submit(_images(0), ids[0])
        b.load_checkpoint(path, pipeline=busy)
    busy.close()
    b.load_checkpoint(path, pipeline=pb)
    pb.submit(_images(s), ids[s])
    lb = []
    for i in range(s, n):
        if i + 1 < n:
            pb.submit(_images(i + 1), ids[i + 1])
        x = pb.get()
        for k, v in got_a[i].items():
            assert torch.equal(x[k], v), (i, k)
        lb.append(b.replay_step(x).cpu().clone())
    pb.close()
    _assert_track(la[s:], lb, a, b)


def test_pipeline_state_dict_is_the_oldest_queued_batch():
    p = _pipe(0)
    s0 = p.state_dict()
    p.submit(_images(0))
    assert p.state_dict() == s0                   # batch 0 not consumed yet
    p.submit(_images(1))
    assert p.state_dict() == s0
    p.get()
    s1 = p.state_dict()
    assert s1 != s0 and isinstance(s1["gen"], bytes)
    p.get()
    assert p.state_dict() not in (s0, s1)         # nothing queued: the current streams
    json.dumps({k: v for k, v in s1.items() if k != "gen"})
    p.close()


def test_teacher_export(tmp_path):
    from vtp_b200 import params as P
    from vtp_b200.model import VTPModel

    a = _trainer(0)
    a.import_state_dict(a.export_state_dict())
    s, t = a.export_state_dict(), a.export_state_dict(teacher=True)
    assert s.keys() == t.keys() and all(torch.equal(s[k], t[k]) for k in s)
    batch = _batch()
    for _ in range(2):
        a.train_step(batch)
    s, t = a.export_state_dict(), a.export_state_dict(teacher=True)
    ema = {}
    for e in a.table:
        if e.teacher and not e.name.startswith("head."):
            ema.update(P.to_reference(e, a.store.tf32(e.name)))
    assert s.keys() == t.keys() and set(ema) < set(t)
    assert any(k.startswith("trunk.") for k in ema) and "visual_proj.weight" in ema
    for k in t:
        if k in ema:
            assert torch.equal(t[k], ema[k]), k
        else:
            assert torch.equal(t[k], s[k]), k
    assert sum(not torch.equal(t[k], s[k]) for k in ema) > len(ema) // 2
    m = VTPModel(a.cfg).cuda()
    m.load_state_dict(t, strict=True)
    out = m.get_last_layer_feature(batch["image"])
    assert torch.isfinite(out["cls_token"].float()).all() and torch.isfinite(out["patch_tokens"].float()).all()


def test_refusals(tmp_path):
    a = _trainer(0)
    a.train_step(_batch())
    path = str(tmp_path / "ck")
    a.save_checkpoint(path)
    other = _trainer(1, K=1024)
    before = _state(other)
    with pytest.raises(ValueError, match=r"wrong shape: param/head\.") as e:
        other.load_checkpoint(path)
    assert "center/dino" in str(e.value) or "(+" in str(e.value)
    _assert_same(before, other)
    # a manifest of a 2-rank job: its RNG streams do not carry over, the rest does
    m = json.load(open(os.path.join(path, "checkpoint.json")))
    m["world_size"] = 2
    json.dump(m, open(os.path.join(path, "checkpoint.json"), "w"))
    b = _trainer(1)
    before = _state(b)
    with pytest.raises(ValueError, match="saved by 2 rank"):
        b.load_checkpoint(path)
    _assert_same(before, b)
    rng = torch.cuda.get_rng_state()
    b.load_checkpoint(path, rng=False)
    assert torch.equal(b.store.p, a.store.p) and torch.equal(b.store.m, a.store.m) and b.step_count == 1
    assert torch.equal(torch.cuda.get_rng_state(), rng)
    with pytest.raises(ValueError, match="no checkpoint.json"):
        b.load_checkpoint(str(tmp_path / "nothing"))


# ------------------------------------------------------------------------------------------------ two ranks
def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _worker(rank, world, port, path, out):
    import torch.distributed as dist

    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    torch.cuda.manual_seed(1000 + rank)              # a different stochastic-depth stream per rank
    dev = f"cuda:{rank}"
    batch = _batch(seed=10 * rank, device=dev)       # this rank's share of the global batch
    a = _trainer(0, device=dev)
    for _ in range(2):
        a.train_step(batch)
    a.save_checkpoint(path)
    saved, rng = _state(a), torch.cuda.get_rng_state(dev)
    la = a.train_step(batch).cpu().clone()
    torch.cuda.manual_seed(7)                        # move the generator away from the saved state
    b = _trainer(1, device=dev)
    b.load_checkpoint(path)
    now = _state(b)
    same = all(v == now[k] if k == "step_count" else torch.equal(v, now[k]) for k, v in saved.items())
    rng_back = torch.equal(torch.cuda.get_rng_state(dev), rng)
    lb = b.train_step(batch).cpu().clone()
    torch.cuda.synchronize()
    p0 = b.store.p.clone()
    dist.broadcast(p0, src=0)
    out[rank] = (same, rng_back, rng.tolist(), la.tolist(), lb.tolist(), rel(b.store.p, a.store.p),
                 rel(b.store.tp, a.store.tp), float((b.store.p - p0).abs().max()))
    dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_rank_resume(tmp_path):
    import torch.multiprocessing as mp

    world, port = 2, _free_port()
    out = mp.Manager().dict()
    path = str(tmp_path / "ck")
    mp.spawn(_worker, args=(world, port, path, out), nprocs=world, join=True)
    assert sorted(os.listdir(path)) == ["checkpoint.json", "rng_rank00.safetensors", "rng_rank01.safetensors",
                                        "trainer.safetensors"]
    for r in range(world):
        same, rng_back, _, la, lb, rp, rtp, pdiff = out[r]
        assert same and rng_back
        assert torch.allclose(torch.tensor(la), torch.tensor(lb), rtol=2e-3, atol=1e-5), (la, lb)
        assert rp < 1e-4 and rtp < 1e-5 and pdiff == 0.0
    assert out[0][2] != out[1][2]                    # each rank got its own stream back
