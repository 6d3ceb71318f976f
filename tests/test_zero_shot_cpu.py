"""Zero-shot host side (vtp_b200/zero_shot.py) without a GPU: prompt fixtures, bucket plan, the rank rule, the CLI."""
import importlib.util
import json
import os

import numpy as np
import pytest
import torch

from vtp_b200 import zero_shot as Z

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
REF = os.environ.get("VTP_REFERENCE_ROOT", "/root/reference")
REF_SCRIPT = os.path.join(REF, "tools", "test_zero_shot_hf.py")
REF_BPE = os.path.join(REF, "tools", "bpe_simple_vocab_16e6.txt.gz")


def prompt_fixture():
    with open(os.path.join(GOLDEN, "zero_shot_prompts.json")) as f:
        meta = json.load(f)
    z = np.load(os.path.join(GOLDEN, "zero_shot_prompts.npz"))
    flat, off = z["ids"].astype(np.int64), z["offsets"]
    ids = np.zeros((len(off) - 1, meta["context_length"]), dtype=np.int64)
    for i in range(len(off) - 1):
        ids[i, :off[i + 1] - off[i]] = flat[off[i]:off[i + 1]]
    return meta, torch.from_numpy(ids)


def rank_rule(logits: np.ndarray, targets: np.ndarray) -> np.ndarray:
    """#{j : l_j ahead of l_t}; NaN above every number, ties (and NaN pairs) to the lower index; C when out of range."""
    B, C = logits.shape
    out = np.full(B, C, dtype=np.int64)
    j = np.arange(C)
    for i, t in enumerate(targets):
        if 0 <= t < C:
            l, lt = logits[i], logits[i, t]
            if np.isnan(lt):
                out[i] = int((np.isnan(l) & (j < t)).sum())
            else:
                out[i] = int((np.isnan(l) | (l > lt) | ((l == lt) & (j < t))).sum())
    return out


def _exec_reference_script():
    """The reference script executed with its heavy imports stubbed out (only its constants are read)."""
    import sys
    import types

    saved = {k: sys.modules.get(k) for k in ("vtp", "vtp.models", "vtp.models.vtp_hf", "vtp.tokenizers")}
    try:
        for k in saved:
            sys.modules[k] = types.ModuleType(k)
        sys.modules["vtp.models.vtp_hf"].VTPConfig = sys.modules["vtp.models.vtp_hf"].VTPModel = object
        sys.modules["vtp.tokenizers"].get_tokenizer = lambda *a, **k: None
        spec = importlib.util.spec_from_file_location("ref_zero_shot_consts", REF_SCRIPT)
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
        return mod
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v


@pytest.mark.skipif(not os.path.exists(REF_SCRIPT), reason="needs the reference's tools/test_zero_shot_hf.py")
def test_ast_prompts_equal_executed_constants():
    pytest.importorskip("tqdm")
    mod = _exec_reference_script()
    names, templates = Z.read_reference_prompts(REF_SCRIPT)
    assert names == list(mod.IMAGENET_CLASSNAMES)
    assert len(templates) == len(mod.OPENAI_IMAGENET_TEMPLATES) == 80
    for fmt, fn in zip(templates, mod.OPENAI_IMAGENET_TEMPLATES):
        assert fmt.format(c="x{y}z") == fn("x{y}z")
    meta, _ = prompt_fixture()
    assert meta["classnames"] == names and meta["templates"] == templates


def test_fixture_templates_give_the_reference_strings():
    meta, ids = prompt_fixture()
    names, templates = meta["classnames"], meta["templates"]
    assert len(names) == 1000 and len(templates) == 80 and ids.shape == (80000, 77)
    assert names.count("missile") == 2 and names.count("sunglasses") == 2     # the reference's duplicates
    texts = [Z.template_fn(t)(c) for c in names for t in templates]
    assert len(set(texts)) < len(texts) == 80000
    assert texts[0] == templates[0].replace("{c}", names[0])
    for t in templates:
        assert t.count("{c}") == 1 and "{" not in t.replace("{c}", "")
    if os.path.exists(REF_SCRIPT):
        pytest.importorskip("tqdm")
        mod = _exec_reference_script()
        assert texts == [fn(c) for c in mod.IMAGENET_CLASSNAMES for fn in mod.OPENAI_IMAGENET_TEMPLATES]


@pytest.mark.skipif(not os.path.exists(REF_BPE), reason="needs the reference vocabulary")
def test_fixture_ids_equal_bpe_tokenizer():
    from vtp_b200.text_tokenizer import BPETokenizer

    meta, ids = prompt_fixture()
    tok = BPETokenizer(bpe_path=REF_BPE, context_length=77)
    texts = [t.format(c=c) for c in meta["classnames"] for t in meta["templates"]]
    assert torch.equal(tok(texts), ids)


def test_bucket_plan_invariants():
    meta, ids = prompt_fixture()
    long_row = torch.arange(1, 78, dtype=torch.int64)[None] % 300 + 1
    long_row[0, 76] = 49407                                   # a 77-token prompt: EOT in the last slot
    ids = torch.cat([ids, long_row])
    eot = Z.eot_positions(ids)
    assert eot.max() == 76
    plan = Z.bucket_plan(eot, 77, max_rows=4096)
    seen = np.concatenate([idx for idx, _ in plan])
    assert np.array_equal(np.sort(seen), np.arange(len(ids)))   # every row exactly once
    rows = 0
    for idx, L in plan:
        assert 1 <= len(idx) <= 4096 and L <= 77
        assert (eot[idx] + 1 <= L).all()
        assert L == min((int(eot[idx].max()) + 8) // 8 * 8, 77)
        rows += len(idx) * L
    assert [L for idx, L in plan if len(ids) - 1 in idx] == [77]
    full = len(ids) * 77
    assert full / rows > 5.0, (rows, full)                      # ~1.13 M token rows instead of 6.16 M
    assert Z.bucket_plan(np.zeros(0, dtype=np.int64), 77) == []


def test_rank_rule_matches_topk_without_boundary_ties():
    g = torch.Generator().manual_seed(0)
    for dtype in (torch.float32, torch.bfloat16):
        logits = (torch.randn(512, 37, generator=g) * 8).to(dtype)
        targets = torch.randint(0, 37, (512,), generator=g)
        r = rank_rule(logits.float().numpy(), targets.numpy())
        for k in (1, 5):
            pred = logits.float().topk(k, 1, True, True)[1]
            hit = (pred == targets[:, None]).any(1).numpy()
            kth = logits.float().topk(k + 1, 1)[0]
            tie = (kth[:, k - 1] == kth[:, k]).numpy()              # a tie across the k boundary: topk may pick either
            assert np.array_equal(hit[~tie], (r < k)[~tie])
        if dtype == torch.bfloat16:
            assert tie.any()


def test_rank_rule_nan_and_out_of_range():
    nan = float("nan")
    logits = np.array([[1.0, nan, 3.0, 3.0], [nan, 2.0, nan, 0.0], [1.0, 2.0, 3.0, 4.0], [0.0, 0.0, 0.0, 0.0]],
                      dtype=np.float32)
    assert rank_rule(logits, np.array([2, 2, 4, -1])).tolist() == [1, 1, 4, 4]
    assert rank_rule(logits, np.array([3, 0, 0, 3])).tolist() == [2, 0, 3, 3]
    sorted_idx = torch.sort(torch.from_numpy(logits[1]), descending=True, stable=True)[1].tolist()
    assert sorted_idx[:2] == [0, 2]                                # torch puts NaN first, the lower index first


def test_cli_flags_defaults_and_fp16():
    ap = Z.build_parser()
    a = ap.parse_args(["--model_path", "m", "--data_path", "d"])
    assert (a.batch_size, a.num_workers, a.device, a.precision) == (128, 8, "cuda:0", "fp32")
    assert a.bpe_path is None and a.prompts is None
    for flag in ("--model_path", "--data_path", "--batch_size", "--num_workers", "--device", "--precision"):
        assert any(flag in act.option_strings for act in ap._actions)
    assert [c for act in ap._actions if "--precision" in act.option_strings for c in act.choices] == ["fp32", "fp16",
                                                                                                       "bf16"]
    with pytest.raises(NotImplementedError):
        Z.main(["--model_path", "m", "--data_path", "d", "--precision", "fp16"])
    with pytest.raises(NotImplementedError):
        Z._mode("fp16")


def test_prompts_json_and_missing_sources(tmp_path, monkeypatch):
    p = tmp_path / "p.json"
    p.write_text(json.dumps({"classnames": ["cat", "dog"], "templates": ["a {c}.", "the {c}!"]}))
    assert Z.load_prompts(str(p)) == (["cat", "dog"], ["a {c}.", "the {c}!"])
    monkeypatch.chdir(tmp_path)
    monkeypatch.delenv("VTP_BPE_PATH", raising=False)
    monkeypatch.setattr(Z, "find_reference_script", lambda bpe_path=None: None)
    with pytest.raises(FileNotFoundError, match="--prompts"):
        Z.load_prompts(None)


def test_reference_script_found_next_to_vocabulary(tmp_path):
    src = "IMAGENET_CLASSNAMES = ('a', 'b{')\nOPENAI_IMAGENET_TEMPLATES = (\n    lambda c: f'x {c} {{y}}.',\n)\n"
    (tmp_path / Z.REFERENCE_SCRIPT).write_text(src)
    (tmp_path / "vocab.txt.gz").write_bytes(b"")
    assert Z.find_reference_script(str(tmp_path / "vocab.txt.gz")) == str(tmp_path / Z.REFERENCE_SCRIPT)
    names, templates = Z.load_prompts(None, str(tmp_path / "vocab.txt.gz"))
    assert names == ["a", "b{"] and templates == ["x {c} {{y}}."]
    assert Z.template_fn(templates[0])("b{") == "x b{ {y}."


def test_accuracy_from_ranks_is_the_reference_formula():
    ranks = np.array([0, 3, 5, 1, 0, 37, 4])
    n = len(ranks)
    assert Z.accuracy_from_ranks(ranks, (1, 5)) == [2.0 / n * 100, 5.0 / n * 100]
