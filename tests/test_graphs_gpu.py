"""VTPModel.enable_cuda_graphs(): captured-graph replays of the inference entry points return exactly what the eager
launches return (same kernels, same order), follow input changes, and are re-captured when the weights change.  Every
graph goes through vtp_b200.graphs.StepGraph: the evaluators capture a graphed model, a replay counts the launches of an
eager call, and a released graph leaves the eager path as it was."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _model(seed=0):
    from oracle.seeded import seeded_state_dict
    from tests.util import load_golden
    from vtp_b200.config import VTPConfig
    from vtp_b200.model import VTPModel

    meta, _ = load_golden("tiny")
    m = VTPModel(VTPConfig(**meta["config"]))
    m.load_state_dict(seeded_state_dict(meta["spec"], seed=seed))
    return m.cuda(), meta


@pytest.mark.parametrize("autocast", [False, True])
def test_graph_replay_equals_eager(autocast):
    from oracle.seeded import seeded_captions, seeded_images, seeded_state_dict

    m, meta = _model()
    x0, x1 = seeded_images(3, 64, 64).cuda(), seeded_images(3, 64, 64, seed=77).cuda()
    ids0, ids1 = seeded_captions(3, 77, 1000).cuda(), seeded_captions(3, 77, 1000, seed=5).cuda()

    def run(x, ids):
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=autocast):
            lat = m.get_reconstruction_latents(x)
            return lat, m.get_latents_decoded_images(lat), m.get_clip_image_feature(x), m.get_clip_text_feature(ids)

    eager = [run(x0, ids0), run(x1, ids1)]
    m.enable_cuda_graphs()
    first = run(x0, ids0)                 # builds the four graphs
    assert len(m._graphs) == 4
    again = run(x1, ids1)                 # pure replays on new input values
    back = run(x0, ids0)
    assert len(m._graphs) == 4
    for got, want in ((first, eager[0]), (again, eager[1]), (back, eager[0])):
        for a, b in zip(got, want):
            assert a.dtype == b.dtype and torch.equal(a, b)
    assert first[0].data_ptr() != back[0].data_ptr()          # outputs are fresh tensors, not the static buffer
    # another batch size -> its own graphs; weight change -> re-capture with the new weights
    small = m.get_reconstruction_latents(x0[:1])
    m.enable_cuda_graphs(False)
    assert torch.equal(small, m.get_reconstruction_latents(x0[:1]))
    m.enable_cuda_graphs()
    m.get_reconstruction_latents(x0)
    m.load_state_dict(seeded_state_dict(meta["spec"], seed=1))
    new_graph = m.get_reconstruction_latents(x0)
    m.enable_cuda_graphs(False)
    assert torch.equal(new_graph, m.get_reconstruction_latents(x0))
    assert not torch.equal(new_graph, eager[0][0].to(new_graph.dtype))


def _launches(fn):
    from vtp_b200 import lib

    l0 = lib.LAUNCHES
    fn()
    return lib.LAUNCHES - l0


def _evaluate(m, batches, targets):
    """Per-image PSNR / SSIM / LPIPS and zero-shot ranks of both evaluators (graph capture on) over the batches."""
    from vtp_b200.lpips import LPIPSMetric
    from vtp_b200.recon_eval import ReconstructionEvaluator
    from vtp_b200.zero_shot import ZeroShotEvaluator

    g = torch.Generator().manual_seed(3)
    clf = torch.nn.functional.normalize(torch.randn(m.visual_proj.weight.shape[0], 11, generator=g), dim=0).cuda()
    rec = ReconstructionEvaluator(m, lpips=LPIPSMetric.random_init(0), precision="bf16", use_graph=True)
    zs = ZeroShotEvaluator(m, clf, precision="bf16", use_graph=True)
    for x, t in zip(batches, targets):
        rec.add(x)
        zs.add(x, t)
    out = dict(rec.per_image(), ranks=zs.ranks(), counts=zs.counts.clone())
    rec.close()
    zs.close()
    return out


def test_evaluators_capture_a_graphed_model():
    """An evaluator captures its whole step on a shape's second batch; the model's entry points called inside that
    capture run their kernels into it instead of replaying their own graphs."""
    from oracle.seeded import seeded_images

    m, _ = _model()
    batches = [seeded_images(3, 64, 64, seed=s).cuda() for s in (1, 2, 3)] + [seeded_images(2, 64, 64, seed=4).cuda()]
    targets = [torch.arange(x.shape[0], device="cuda") * 5 % 11 for x in batches]
    want = _evaluate(m, batches, targets)
    m.enable_cuda_graphs()
    got = _evaluate(m, batches, targets)
    assert len(m._graphs) == 6      # per batch shape: latents, decode and the image feature, from the eager batches
    for k, v in want.items():
        assert torch.equal(got[k], v), k


def test_replay_counts_the_launches_of_an_eager_call():
    from oracle.seeded import seeded_images
    from vtp_b200.recon_eval import ReconstructionEvaluator

    m, _ = _model()
    x = seeded_images(3, 64, 64).cuda()
    m.get_reconstruction_latents(x)                           # packs the weights
    eager = _launches(lambda: m.get_reconstruction_latents(x))
    m.enable_cuda_graphs()
    m.get_reconstruction_latents(x)                           # warm-up and capture
    assert eager > 0 and _launches(lambda: m.get_reconstruction_latents(x)) == eager
    m.enable_cuda_graphs(False)
    evs = [ReconstructionEvaluator(m, precision="bf16", use_graph=g) for g in (False, True)]
    for _ in range(2):                                        # packs, then the capture
        for ev in evs:
            ev.add(x)
    counts = [_launches(lambda: ev.add(x)) for ev in evs]
    assert counts[0] > 0 and counts[1] == counts[0]
    for ev in evs:
        ev.close()


def test_release_twice_and_eager_after_release():
    from oracle.seeded import seeded_images
    from vtp_b200.recon_eval import ReconstructionEvaluator

    m, _ = _model()
    x = seeded_images(3, 64, 64).cuda()
    want = m.get_reconstruction_latents(x)
    m.enable_cuda_graphs()
    assert torch.equal(m.get_reconstruction_latents(x), want)
    (_, graph, _, _), = m._graphs.values()
    m.enable_cuda_graphs(False)
    assert graph.graph is None and not m._graphs
    graph.release()
    assert torch.equal(m.get_reconstruction_latents(x), want)
    ev = ReconstructionEvaluator(m, precision="bf16", use_graph=True)
    for _ in range(3):
        ev.add(x)
    (st,) = ev._steps.values()
    assert st.graph.graph is not None
    ev.close()
    ev.close()
    assert st.graph.graph is None
    eager = ReconstructionEvaluator(m, precision="bf16", use_graph=False)
    for _ in range(3):
        eager.add(x)
    for k, v in eager.per_image().items():
        assert torch.equal(ev.per_image()[k], v), k
    eager.close()
