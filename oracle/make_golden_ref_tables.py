"""Record what the reference computes for the host-side pieces restated in vtp_b200 (run where the reference is importable):

  * caption tokenizer: the reference's `SimpleTokenizer` on a PREFIX of its BPE vocabulary (the first N_MERGES merges, stored
    as tests/golden/bpe_prefix.txt.gz — the whole file is 1.3 MB): vocabulary layout, ids of every caption of the test corpus
    at several context lengths, decodings, and the no-lower-casing + extra-special-token variant;
  * stochastic depth: `get_branges_scales` (layers/block.py:20-118) single process and on 2 gloo ranks;
  * `CosineScheduler` (utils/text_utils.py) over every iteration of the test cases.

Usage:  python -m oracle.make_golden_ref_tables      (writes tests/golden/bpe_prefix.txt.gz, ref_tables.json, tokenizer_ids.npz)
"""
from __future__ import annotations

import gzip
import importlib.util
import json
import os
import socket
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden")
N_MERGES = 16000

from oracle import ref_harness as rh  # noqa: E402
from tests.test_tokenizer_cpu import CORPUS, LENGTHS, full_corpus  # noqa: E402

DROP_CASES = [(8, 0.3), (5, 0.5), (3, 0.9), (256, 0.25), (1, 0.5)]
DROP_CASES_DP = [(8, 0.3), (5, 0.5), (3, 0.9), (16, 0.1)]
COSINE_CASES = [dict(base_value=1e-3, final_value=1e-6, total_iters=50, warmup_iters=5, start_warmup_value=1e-7, freeze_iters=0),
                dict(base_value=0.994, final_value=1.0, total_iters=20),
                dict(base_value=0.04, final_value=0.2, total_iters=12, warmup_iters=3, start_warmup_value=0.0, freeze_iters=2)]


def _drop_worker(rank, world, port, out):
    import torch.distributed as dist

    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    rh.import_reference()
    import vtp.models.layers.block as blk

    res = []
    for b, ratio in DROP_CASES_DP:
        br, scale = blk.get_branges_scales(torch.zeros(b, 2, 4), ratio)
        res.append([b, ratio, int(br.numel()), float(scale)])
    out[rank] = res
    dist.destroy_process_group()


def main():
    rh.import_reference()
    # ---- tokenizer on a vocabulary prefix
    src = os.path.join(rh.REF_ROOT, "tools", "bpe_simple_vocab_16e6.txt.gz")
    lines = gzip.open(src).read().decode("utf-8").split("\n")
    bpe = os.path.join(GOLDEN, "bpe_prefix.txt.gz")
    with gzip.GzipFile(bpe, "wb", mtime=0) as f:
        f.write("\n".join(lines[: N_MERGES + 1]).encode("utf-8"))
    spec = importlib.util.spec_from_file_location("_ref_tt", os.path.join(rh.REF_ROOT, "vtp", "tokenizers", "text_tokenizer.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    ref = mod.SimpleTokenizer(bpe)
    corpus = full_corpus()
    enc = [ref.encode(t) for t in corpus]
    arrays = {"enc_flat": np.array([i for e in enc for i in e], dtype=np.int32),
              "enc_len": np.array([len(e) for e in enc], dtype=np.int32)}
    for L in LENGTHS:
        arrays[f"ids_{L}"] = ref(corpus, L).numpy().astype(np.int32)
    arrays["ids_one"] = ref("one caption").numpy().astype(np.int32)
    arrays["decoded"] = np.array([ref.decode(e) for e in enc])
    r2 = mod.SimpleTokenizer(bpe, clean="whitespace", additional_special_tokens=["<mask>"])
    extra = corpus + ["Keep CASE <mask> <Mask> <start_of_text>"]
    arrays["ids_ws_mask"] = r2(extra).numpy().astype(np.int32)
    np.savez_compressed(os.path.join(GOLDEN, "tokenizer_ids.npz"), **arrays)
    tables = {"tokenizer": {"n_merges": N_MERGES, "vocab_size": ref.vocab_size, "sot": ref.sot_token_id,
                            "eot": ref.eot_token_id, "special_ids": list(ref.all_special_ids),
                            "context_length": ref.context_length, "vocab_size_ws_mask": r2.vocab_size}}
    # ---- stochastic depth allocation
    import vtp.models.layers.block as blk

    single = []
    for b, ratio in DROP_CASES:
        br, scale = blk.get_branges_scales(torch.zeros(b, 2, 4), ratio)
        single.append([b, ratio, int(br.numel()), float(scale)])
    import torch.multiprocessing as mp

    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    out = mp.Manager().dict()
    mp.spawn(_drop_worker, args=(2, port, out), nprocs=2, join=True)
    tables["drop_plan"] = {"single": single, "dp2": {str(r): out[r] for r in (0, 1)}}
    # ---- cosine schedule
    from vtp.models.utils.text_utils import CosineScheduler

    tables["cosine"] = [{"kwargs": kw, "values": [float(CosineScheduler(**kw)[i]) for i in range(kw["total_iters"] + 3)]}
                        for kw in COSINE_CASES]
    with open(os.path.join(GOLDEN, "ref_tables.json"), "w") as f:
        json.dump(tables, f, separators=(",", ":"))
        f.write("\n")


if __name__ == "__main__":
    main()
