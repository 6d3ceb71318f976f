"""Caption tokenizer (vtp_b200/text_tokenizer.py, SURVEY.md §8(f)4) — CPU tests.

  * against what the reference `SimpleTokenizer` (vtp/tokenizers/text_tokenizer.py:144-295) computed on the first 16 000
    merges of its own vocabulary file (tests/golden/bpe_prefix.txt.gz, tokenizer_ids.npz, ref_tables.json; recorded by
    oracle/make_golden_ref_tables.py): identical vocabulary layout, identical ids for every caption of a corpus built to
    hit the pattern's branches, identical truncation and decoding;
  * self-contained cases on a tiny synthetic vocabulary (written to a temp dir): merge order, end-of-word variants,
    special tokens, truncation rule, errors."""
import gzip
import json
import os
import random

import numpy as np
import pytest
import torch

from vtp_b200.text_tokenizer import BPETokenizer, find_bpe_file, get_tokenizer

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
BPE_PREFIX = os.path.join(GOLDEN, "bpe_prefix.txt.gz")
LENGTHS = (77, 8, 16, 200)

CORPUS = [
    "a photo of a cat", "A Photo of a CAT!!!", "  multiple   spaces\tand\nnewlines ",
    "it's the dog's ball, they've won; I'm here, we'll go, he'd say, don't", "'s't're've'm'll'd", "''''",
    "naïve café déjà vu — “quotes” ‘single’ … ellipsis", "日本語のテキスト と 中文文本 and한국어", "emoji 😀😃 🤖👍🏽 flags 🇩🇪",
    "numbers 1234567890 3.14159 1e-5 ½ ²", "&amp;lt;b&amp;gt; html &amp; entities &lt;i&gt; &#39;x&#39;",
    "<start_of_text> literal specials <end_of_text> inside", "<START_OF_TEXT> upper special", "", "   ", "x", "a" * 300,
    "word " * 200, "supercalifragilisticexpialidocious antidisestablishmentarianism",
    "e-mail: someone@example.com, http://example.com/path?query=1&b=2", "tabs\tand\x00control\x07chars",
    "mixed123abc456 under_score-dash", "ÀÉÎÕÜ ßẞ ǅ İi", "𝔘𝔫𝔦𝔠𝔬𝔡𝔢 math 𝟘𝟙𝟚", "！？。、", "á combining ë",
]


def full_corpus():
    rng = random.Random(0)
    alphabet = "abcdefghijklmnopqrstuvwxyz  ABC.,!?'0123456789-éüñ日本😀"
    return CORPUS + ["".join(rng.choice(alphabet) for _ in range(rng.randint(1, 120))) for _ in range(400)]


def test_token_ids_equal_the_live_reference():
    """(The name is historical: the comparison runs against what the reference recorded, see the module docstring.)"""
    ref = json.load(open(os.path.join(GOLDEN, "ref_tables.json"), encoding="utf-8"))["tokenizer"]
    g = np.load(os.path.join(GOLDEN, "tokenizer_ids.npz"))
    ours = BPETokenizer(BPE_PREFIX)
    assert (ours.vocab_size, ours.sot_token_id, ours.eot_token_id, list(ours.all_special_ids), ours.context_length) == \
           (ref["vocab_size"], ref["sot"], ref["eot"], ref["special_ids"], ref["context_length"])
    corpus = full_corpus()
    offs = np.concatenate([[0], np.cumsum(g["enc_len"])])
    for i, text in enumerate(corpus):
        a = ours.encode(text)
        assert a == g["enc_flat"][offs[i]:offs[i + 1]].tolist(), text
        assert ours.decode(a) == str(g["decoded"][i])
    for L in LENGTHS:                           # padding, exact fit, truncation (last slot becomes <end_of_text>)
        x = ours(corpus, L)
        assert x.dtype == torch.long and torch.equal(x, torch.from_numpy(g[f"ids_{L}"]).long())
    assert torch.equal(ours("one caption"), torch.from_numpy(g["ids_one"]).long())
    # second call: served from the caption cache, same ids
    assert torch.equal(ours(corpus), torch.from_numpy(g["ids_77"]).long())
    # no lower-casing + an extra special token (case-sensitive cache hit of specials, as upstream)
    o2 = BPETokenizer(BPE_PREFIX, clean="whitespace", additional_special_tokens=["<mask>"])
    extra = corpus + ["Keep CASE <mask> <Mask> <start_of_text>"]
    assert torch.equal(o2(extra), torch.from_numpy(g["ids_ws_mask"]).long())
    assert o2.vocab_size == ref["vocab_size_ws_mask"] == ours.vocab_size + 1
    assert get_tokenizer(bpe_path=BPE_PREFIX, context_length=32)("a cat").shape == (1, 32)


def _tiny_vocab(tmp_path):
    """header line + five merges: 't h', 'th e</w>', 'c a', 'ca t</w>', 'a t</w>' (the last can never apply after 'c a')."""
    p = tmp_path / "tiny_bpe.txt.gz"
    with gzip.open(p, "wb") as f:
        f.write('"version"\nt h\nth e</w>\nc a\nca t</w>\na t</w>\n'.encode("utf-8"))
    return str(p)


def test_merge_order_and_layout_on_a_synthetic_vocabulary(tmp_path):
    tok = BPETokenizer(_tiny_vocab(tmp_path), context_length=8)
    # layout: 256 byte symbols, 256 end-of-word variants, merges in file order (a trailing empty line yields one more,
    # empty, entry exactly as upstream's split('\n')), then the two special tokens
    assert tok.encoder["th"] == 512 and tok.encoder["the</w>"] == 513 and tok.encoder["cat</w>"] == 515
    assert tok.sot_token_id == tok.vocab_size - 2 and tok.eot_token_id == tok.vocab_size - 1
    b = lambda ch: tok.encoder[ch]
    assert tok.encode("the") == [513]                                   # t h -> th ; th e</w> -> the</w>
    assert tok.encode("The  cat") == [513, 515]                         # lower-cased, whitespace collapsed
    assert tok.encode("that") == [512, tok.encoder["at</w>"]]           # 't h' (rank 0) before 'a t</w>' (rank 4)
    assert tok.encode("tht") == [512, b("t</w>")]                       # no merge for (th, t</w>)
    assert tok.encode("ththe") == [512, 513]                            # every occurrence of the best pair merges per round
    assert tok.encode("é") == [b("Ã"), b("©") + 256]                    # two UTF-8 bytes, the last one end-of-word
    assert tok.encode("<end_of_text>") == [tok.eot_token_id]
    assert tok.decode(tok.encode("the cat é")) == "the cat é "
    out = tok(["the", "the cat the cat the cat the cat", ""])
    sot, eot = tok.sot_token_id, tok.eot_token_id
    assert out.tolist() == [[sot, 513, eot, 0, 0, 0, 0, 0],
                            [sot, 513, 515, 513, 515, 513, 515, eot],    # cut to 8, last slot = end token
                            [sot, eot, 0, 0, 0, 0, 0, 0]]
    assert tok(["the"], context_length=2).tolist() == [[sot, eot]]


def test_vocabulary_lookup_and_errors(tmp_path, monkeypatch):
    with pytest.raises(FileNotFoundError):
        BPETokenizer(str(tmp_path / "missing.txt.gz"))
    monkeypatch.setenv("VTP_BPE_PATH", _tiny_vocab(tmp_path))
    assert find_bpe_file() == os.path.abspath(_tiny_vocab(tmp_path))
    assert BPETokenizer().encode("the") == [513]
    with pytest.raises(AssertionError):
        BPETokenizer(context_length=None)("x")
