"""The parameter table (vtp_b200/params.py) against VTPModel's state dict, the trainer's flat store, the inference
packer and the memory model — host logic, no GPU."""
import math

import pytest
import torch

from oracle.seeded import seeded_state_dict
from vtp_b200 import memory
from vtp_b200 import params as P
from vtp_b200.config import preset
from vtp_b200.engine import BF, F32, Lin
from vtp_b200.model import VTPModel
from vtp_b200.rope import rope_periods
from vtp_b200.train import ParamStore, store_tower

PRESETS = {"tiny": ("tiny", {}), "small": ("small", {}), "large": ("large", {}),
           "swiglu64": ("tiny", dict(vision_ffn_layer="swiglu64", decoder_ffn_layer="swiglu64"))}
HEAD = (512, 256, 64)   # DINO head (out_dim, hidden, bottleneck)


def config(name, shallow=False):
    base, over = PRESETS[name]
    if shallow:   # the preset's widths at one block per tower and a short vocabulary: small enough for CPU tensors
        over = dict(over, vision_depth=1, decoder_depth=1, text_depth=1, text_vocab_size=2048)
    return preset(base, **over)


def model_shapes(cfg):
    with torch.device("meta"):
        m = VTPModel(cfg)
    return m, {k: tuple(v.shape) for k, v in m.state_dict().items() if not k.endswith("rope_embed.periods")}


def seeded(cfg):
    sd = seeded_state_dict({k: list(s) for k, s in model_shapes(cfg)[1].items()}, seed=0)
    K, hh, hb = HEAD
    D = cfg.vision_embed_dim
    hsd = seeded_state_dict({"mlp.0.weight": [hh, D], "mlp.0.bias": [hh], "mlp.2.weight": [hh, hh], "mlp.2.bias": [hh],
                             "mlp.4.weight": [hb, hh], "mlp.4.bias": [hb], "last_layer.weight_g": [K, 1],
                             "last_layer.weight_v": [K, hb]}, seed=3)
    return sd, hsd


def flat_store(cfg, sd, hsd):
    """The trainer's ParamStore on the host, filled by its import; the bf16 copy as sync_compute_copies makes it."""
    entries = P.table(cfg, HEAD)
    st = ParamStore("cpu")
    for e in entries:
        st.add(e.name, e.shape, e.decay, e.teacher)
    st.finalize()
    P.import_reference(entries, st.f32, sd, hsd)
    st.pb.copy_(st.p.to(BF))
    return entries, st


def same_bits(a, b):
    if a.dtype != b.dtype or a.shape != b.shape:
        return False
    as_int = torch.int16 if a.dtype == BF else torch.int32
    return torch.equal(a.contiguous().view(as_int), b.contiguous().view(as_int))


@pytest.mark.parametrize("name", PRESETS)
def test_table_consumes_every_reference_key_once(name):
    cfg = config(name)
    refs = [(k, e.ref_shape) for e in P.table(cfg) for k in e.ref]
    assert len(refs) == len({k for k, _ in refs})
    assert dict(refs) == model_shapes(cfg)[1]
    for e in P.table(cfg, HEAD):
        assert math.prod(e.shape) == len(e.ref) * math.prod(e.ref_shape), e.name


@pytest.mark.parametrize("name", PRESETS)
def test_export_inverts_import(name):
    cfg = config(name, shallow=True)
    sd, hsd = seeded(cfg)
    entries, st = flat_store(cfg, sd, hsd)
    out = P.export_reference(entries, st.f32)
    want = {**sd, **hsd}
    assert out.keys() == want.keys()
    for k, v in want.items():
        assert same_bits(out[k], v), k
    # the weight_norm parametrization's spelling of the head's last layer imports to the same flat buffer
    _, st2 = flat_store(cfg, sd, {P._WEIGHT_NORM.get(k, k): v for k, v in hsd.items()})
    assert same_bits(st2.p, st.p)


@pytest.mark.parametrize("name", PRESETS)
def test_inference_packing_matches_the_trainer_layout(name):
    """bf16-mode packing of a state dict and the trainer's views of the same state dict give the same tensors.  The
    weights are bf16-representable, so autocast's bias rounding in the inference packer changes no bit."""
    cfg = config(name, shallow=True)
    sd, hsd = seeded(cfg)
    sd = {k: v.to(BF).to(F32) for k, v in sd.items()}
    _, st = flat_store(cfg, sd, hsd)
    sd.update({k: rope_periods(64) for k in ("trunk.rope_embed.periods", "pixel_decoder.rope_embed.periods")})

    def check(a, b, what):
        if a is None or b is None:
            assert a is None and b is None, what
        elif isinstance(a, Lin):
            assert (a.N, a.K) == (b.N, b.K), what
            check(a.w, b.w, what)
            check(a.b, b.b, what)
        elif isinstance(a, torch.Tensor):
            assert same_bits(a, b), what
        else:
            assert a == b, what

    for tower in ("trunk", "decoder", "text"):
        inf = P.pack_tower(sd, cfg, tower, "bf16")
        trn = store_tower(cfg, st.offset, tower, st.bf16, st.f32)
        for f in ("D", "heads", "norm", "eps", "stream_bf16", "prefix", "ffn"):
            check(getattr(inf, f), getattr(trn, f), f)
        assert len(inf.blocks) == len(trn.blocks)
        for i, (a, b) in enumerate(zip(inf.blocks, trn.blocks)):
            for f in ("n1_w", "n1_b", "qkv", "proj", "n2_w", "n2_b", "fc1", "fc2", "hidden"):
                check(getattr(a, f), getattr(b, f), f"{tower}.blocks.{i}.{f}")
        check(inf.norm_w, trn.norm_w, "norm_w")
        check(inf.norm_b, trn.norm_b, "norm_b")
        for k, v in inf.extra.items():
            check(v, trn.extra[k], k)


@pytest.mark.parametrize("name", PRESETS)
def test_param_count_is_the_table(name):
    cfg = config(name)
    m, _ = model_shapes(cfg)
    K, hh, hb = 65536, 2048, 256
    head = hh * cfg.vision_embed_dim + hh + hh * hh + hh + hb * hh + hb + K * hb + K
    teacher = sum(p.numel() for n, p in m.named_parameters() if n.startswith(("trunk.", "visual_proj.")))
    n = memory.param_count(cfg)
    assert n["total"] == sum(math.prod(e.shape) for e in P.table(cfg, (K, hh, hb)))
    assert n["total"] == sum(p.numel() for p in m.parameters()) + head
    assert n["teacher"] == teacher + head


@pytest.mark.parametrize("lpips", [True, False])
def test_batch_and_image_groups_at_the_benchmark_defaults(lpips):
    """bench.py's batch and SSL / reconstruction image groups for every preset (256 images asked, K = 65 536)."""
    want = {"tiny": (256, (0, 0)), "small": (256, (0, 0)), "base": (256, (128, 0)), "large": (128, (64, 64))}
    for name, (B, chunks) in want.items():
        assert memory.fit_batch(preset(name), 256, head_out_dim=65536, lpips=lpips) == B, name
        assert memory.suggest_chunks(preset(name), B, head_out_dim=65536, lpips=lpips) == chunks, name
