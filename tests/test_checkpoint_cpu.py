"""The training-checkpoint format (vtp_b200/checkpoint.py) on its own, with CPU tensors and no trainer: write / read
round trip, refusal of incomplete or mismatched checkpoints with messages that name the offending entries, and the
JSON round trip of an input pipeline's NumPy RNG states."""
import json
import os

import numpy as np
import pytest
import torch

from vtp_b200 import checkpoint as C
from vtp_b200 import params as P
from vtp_b200.config import preset

K = 512


def _spec():
    return C.state_spec(P.table(preset("tiny"), (K, 256, 64)), K)


def _tensors(spec, seed=0):
    g = torch.Generator().manual_seed(seed)
    return {n: torch.randn(s, generator=g) for n, s in spec.items()}


def _pipeline_state(seed=3):
    rng, photo = np.random.default_rng(seed), np.random.default_rng([seed, 1])
    rng.random(17), photo.integers(0, 24, 5)          # somewhere inside the streams
    return {"rng": rng.bit_generator.state, "photo_rng": photo.bit_generator.state, "gen": bytes(range(16))}


def _save(path, tensors, step=7, pipeline=None):
    C.save(str(path), tensors, step=step, cuda_rng=torch.arange(16, dtype=torch.uint8), pipeline=pipeline,
           config={"model": {"vision_embed_dim": 128}, "train": {"head_out_dim": K}})


def test_spec_covers_the_table():
    table = P.table(preset("tiny"), (K, 256, 64))
    spec = _spec()
    n_teacher = sum(e.teacher for e in table)
    assert len(spec) == 3 * len(table) + n_teacher + 3
    assert spec["param/head.last_v"] == (K, 64) and spec["teacher/trunk.patch.w"] == (128, 768)
    assert "teacher/decoder.proj_in.w" not in spec and "teacher/text.tok_emb" not in spec
    assert spec["center/dino"] == spec["center/ibot"] == (K,)
    # size of the state file: 12 B per parameter, 4 more per teacher parameter, the centres, the step (+ the header)
    from vtp_b200.memory import param_count
    n = param_count(preset("tiny"), K, 256, 64)
    assert sum(int(np.prod(s)) for s in spec.values()) * 4 == n["total"] * 12 + n["teacher"] * 4 + 2 * K * 4 + 12


def test_round_trip(tmp_path):
    from safetensors.torch import load_file

    spec = _spec()
    t = _tensors(spec)
    path = tmp_path / "ck"
    pipe = _pipeline_state()
    _save(path, t, step=7, pipeline=pipe)
    assert sorted(os.listdir(path)) == [C.MANIFEST, C.rng_file(0), C.STATE_FILE]
    assert not os.path.exists(str(path) + ".tmp")
    ck = C.load(str(path), spec, pipeline=True)
    assert ck.step == 7 and ck.world_size == 1
    assert set(ck.names) == set(spec)
    for n, v in t.items():
        assert torch.equal(ck.tensor(n), v), n
    assert torch.equal(ck.cuda_rng, torch.arange(16, dtype=torch.uint8))
    assert ck.pipeline == pipe
    # the files are plain safetensors
    assert all(torch.equal(v, t[n]) for n, v in load_file(os.path.join(path, C.STATE_FILE)).items())
    m = json.load(open(os.path.join(path, C.MANIFEST)))
    assert m["files"][C.STATE_FILE] == os.path.getsize(os.path.join(path, C.STATE_FILE))
    assert m["config"]["train"]["head_out_dim"] == K
    # views of one flat buffer (how the trainer hands them over) are written one by one
    flat = torch.arange(10, dtype=torch.float32)
    _save(tmp_path / "views", {"a": flat[0:4], "b": flat[4:10].view(2, 3)})
    ck = C.load(str(tmp_path / "views"), {"a": (4,), "b": (2, 3)})
    assert torch.equal(ck.tensor("a"), flat[:4]) and torch.equal(ck.tensor("b"), flat[4:].view(2, 3))
    assert ck.pipeline is None
    with pytest.raises(ValueError, match="without an input pipeline"):
        C.load(str(tmp_path / "views"), {"a": (4,), "b": (2, 3)}, pipeline=True)


def test_overwrite_replaces_the_previous_checkpoint(tmp_path):
    spec = _spec()
    path = tmp_path / "ck"
    _save(path, _tensors(spec, 0), step=3)
    t1 = _tensors(spec, 1)
    _save(path, t1, step=4)
    ck = C.load(str(path), spec)
    assert ck.step == 4 and torch.equal(ck.tensor("param/trunk.cls"), t1["param/trunk.cls"])
    assert sorted(os.listdir(tmp_path)) == ["ck"]


def test_incomplete_checkpoints_are_refused(tmp_path):
    spec = _spec()
    t = _tensors(spec)
    path = tmp_path / "ck"
    _save(path, t)
    # a save that stopped before the manifest: only the .tmp directory, which is not a checkpoint ...
    tmp = str(path) + ".tmp"
    os.makedirs(tmp)
    with open(os.path.join(tmp, C.STATE_FILE), "wb") as f:
        f.write(b"\0" * 100)
    with pytest.raises(ValueError, match="no checkpoint.json"):
        C.load(tmp, spec)
    # ... is ignored by a load of the checkpoint of that name, and cleared by the next save
    assert torch.equal(C.load(str(path), spec).tensor("center/dino"), t["center/dino"])
    _save(path, t, step=8)
    assert not os.path.exists(tmp) and C.load(str(path), spec).step == 8
    # a directory without a manifest
    os.remove(os.path.join(path, C.MANIFEST))
    with pytest.raises(ValueError, match="no checkpoint.json"):
        C.load(str(path), spec)
    with pytest.raises(ValueError, match="no checkpoint.json"):
        C.load(str(tmp_path / "nowhere"), spec)
    # a truncated file
    _save(path, t)
    fn = os.path.join(path, C.STATE_FILE)
    size = os.path.getsize(fn)
    with open(fn, "r+b") as f:
        f.truncate(size - 4)
    with pytest.raises(ValueError, match=f"{C.STATE_FILE} \\({size - 4} B, manifest {size} B\\)"):
        C.load(str(path), spec)
    # a missing RNG file
    _save(path, t)
    os.remove(os.path.join(path, C.rng_file(0)))
    with pytest.raises(ValueError, match="rng_rank00.safetensors \\(missing"):
        C.load(str(path), spec)


def test_mismatched_names_are_named(tmp_path):
    spec = _spec()
    path = tmp_path / "ck"
    _save(path, _tensors(spec))
    # another head_out_dim: wrong shapes, and the head entries come first
    other = C.state_spec(P.table(preset("tiny"), (1024, 256, 64)), 1024)
    with pytest.raises(ValueError, match=r"wrong shape: param/head\.last_v F32\[512, 64\] \(expected F32\[1024, 64\]\), "
                                         r"param/head\.last_g") as e:
        C.load(str(path), other)
    assert "(+" in str(e.value) and "missing" not in str(e.value) and "unexpected" not in str(e.value)
    # missing and unexpected names
    fewer = {n: s for n, s in spec.items() if n != "exp_avg/trunk.cls"}
    more = dict(spec, **{"param/extra.w": (3, 4)})
    with pytest.raises(ValueError, match=r"unexpected: exp_avg/trunk\.cls$"):
        C.load(str(path), fewer)
    with pytest.raises(ValueError, match=r"missing: param/extra\.w$"):
        C.load(str(path), more)
    # another preset altogether
    with pytest.raises(ValueError, match="wrong shape: param/trunk.patch.w") as e:
        C.load(str(path), C.state_spec(P.table(preset("small"), (K, 256, 64)), K))
    assert "missing" in str(e.value) and "unexpected" not in str(e.value)


def test_world_size_and_rng(tmp_path):
    spec = _spec()
    path = tmp_path / "ck"
    _save(path, _tensors(spec), pipeline=_pipeline_state())
    m = json.load(open(os.path.join(path, C.MANIFEST)))
    m["world_size"] = 2
    with open(os.path.join(path, C.MANIFEST), "w") as f:
        json.dump(m, f)
    with pytest.raises(ValueError, match="saved by 2 rank"):
        C.load(str(path), spec)
    ck = C.load(str(path), spec, rng=False)
    assert ck.cuda_rng is None and ck.pipeline is None and ck.world_size == 2
    with pytest.raises(ValueError, match="rng=True"):
        C.load(str(path), spec, rng=False, pipeline=True)


def test_pipeline_numpy_states_survive_json(tmp_path):
    """The NumPy bit-generator states go into the RNG file's JSON metadata (128-bit PCG64 integers included) and draw
    the same numbers afterwards; the CUDA generator state comes back as the same bytes."""
    state = _pipeline_state(seed=11)
    a = np.random.default_rng()
    a.bit_generator.state = state["rng"]
    expect = a.random(8), a.uniform(0.3, 1.0, 4)
    _save(tmp_path / "ck", _tensors(_spec()), pipeline=state)
    back = C.load(str(tmp_path / "ck"), _spec(), pipeline=True).pipeline
    assert back == state and isinstance(back["gen"], bytes)
    b = np.random.default_rng(0)
    b.bit_generator.state = back["rng"]
    got = b.random(8), b.uniform(0.3, 1.0, 4)
    assert all(np.array_equal(x, y) for x, y in zip(expect, got))
    assert state["rng"]["state"]["state"] > 2 ** 64      # the full 128-bit state, not a float approximation
