"""Device byte-level BPE tokenizer on the H100: the kernels' ids against the Hugging Face tokenizer call for the RoBERTa,
ModernBERT and EuroBERT shapes, and the classifier's text path through it against the host-tokenized path, bit for bit."""
import numpy as np
import pytest
import torch

import bpe_corpus as bc
import tokenizer_corpus as tc

pytestmark = pytest.mark.gpu


def _batch(B: int, max_length: int) -> list:
    texts = bc.BPE_TRAPS + tc.random_texts(64, seed=B + max_length) + ["a" * 1_000_000, "x " + "é" * 300_000 + " y"]
    if max_length == 8192:
        texts.append(" ".join(tc.random_texts(400, seed=5)))           # past 8192 tokens: truncated
    return (texts * (B // len(texts) + 1))[:B] if B > len(texts) else texts[-B:] if B < 8 else texts[:B]


@pytest.mark.parametrize("kind", bc.KINDS)
def test_device_ids_equal_hf(cabi, kind):
    tok = bc.make_bpe(kind, 30000)
    dev, why = cabi.BPETokenizer.from_hf(tok)
    assert dev is not None, why
    for max_length in (8, 128, 512, 8192):
        for B in (1, 7, 512, 1024):
            texts = _batch(B, max_length)
            ids, mask, tt = dev(texts, max_length)
            torch.cuda.synchronize()
            ref = tok(texts, max_length=max_length, truncation=True, padding=True, return_tensors="pt")
            assert torch.equal(ids.cpu(), ref["input_ids"].to(torch.int32)), (kind, max_length, B)
            assert torch.equal(mask.cpu(), ref["attention_mask"].to(torch.int32))
            assert tt is None and "token_type_ids" not in ref
    assert dev(["ok", "bad \ud800 surrogate"], 16) is None                 # no UTF-8 form: the caller's host path decides


def test_handmade_merges_on_the_device(cabi):
    """ties, runs of one symbol, a non-monotone rank order and ignore_merges, as the CPU shim runs them"""
    for tok, texts in (
            (bc.make_handmade("roberta", [("a", "a"), ("aa", "a"), ("b", "b"), ("bb", "bb")]),
             ["a" * n for n in range(1, 12)] + ["aaaa aaa", "abababa"]),
            (bc.make_handmade("eurobert", [("p", "qr"), ("pq", "r"), ("q", "r"), ("p", "q"), ("pqr", "pqr")]),
             ["pqr", "pqrpqr", "rpqr", "qrp", "pqpqr"]),
            (bc.make_handmade("eurobert", [("e", "n"), ("en", "d")], extra=["endoftext", "Ġendoftext"], ignore_merges=True),
             ["endoftext", "x endoftext endof end"])):
        dev, why = cabi.BPETokenizer.from_hf(tok)
        assert dev is not None, why
        ids, mask, _ = dev(texts, 32)
        ref = tok(texts, max_length=32, truncation=True, padding=True, return_tensors="pt")
        assert torch.equal(ids.cpu(), ref["input_ids"].to(torch.int32)) and torch.equal(mask.cpu(), ref["attention_mask"].to(torch.int32))


def _checkpoint(tmp_path, kind: str) -> str:
    from transformers import (EuroBertConfig, EuroBertModel, ModernBertConfig, ModernBertModel, RobertaConfig,
                              RobertaModel)
    torch.manual_seed(11)
    d = str(tmp_path / kind)
    tok = bc.make_bpe({"roberta": "roberta", "modernbert": "modernbert", "eurobert": "eurobert"}[kind])
    n = len(tok)
    if kind == "roberta":
        m = RobertaModel(RobertaConfig(vocab_size=n, hidden_size=128, num_hidden_layers=2, num_attention_heads=2,
                                       intermediate_size=256, max_position_embeddings=514, pad_token_id=tok.pad_token_id))
    elif kind == "modernbert":
        m = ModernBertModel(ModernBertConfig(vocab_size=n, hidden_size=128, num_hidden_layers=2, num_attention_heads=2,
                                             intermediate_size=64, local_attention=16, max_position_embeddings=8192,
                                             pad_token_id=tok.pad_token_id, cls_token_id=tok.cls_token_id,
                                             sep_token_id=tok.sep_token_id, bos_token_id=tok.cls_token_id,
                                             eos_token_id=tok.sep_token_id))
    else:
        m = EuroBertModel(EuroBertConfig(vocab_size=n, hidden_size=256, num_hidden_layers=2, num_attention_heads=4,
                                         num_key_value_heads=2, intermediate_size=512, max_position_embeddings=8192,
                                         rope_parameters={"rope_type": "default", "rope_theta": 250000.0},
                                         bos_token_id=tok.bos_token_id, eos_token_id=tok.eos_token_id,
                                         pad_token_id=tok.pad_token_id))
    m.eval().save_pretrained(d)
    tok.save_pretrained(d)
    return d


@pytest.mark.parametrize("kind,max_length", [("roberta", 512), ("modernbert", 512), ("modernbert", 8192), ("eurobert", 512)])
def test_classifier_text_path_is_bitwise_the_host_path(cabi, tmp_path, kind, max_length):
    import adaptive_classifier_b200 as acb
    config = {"max_length": max_length} if max_length != 512 else {}
    clf = acb.AdaptiveClassifier(_checkpoint(tmp_path, kind), device="cuda", config=config)
    assert isinstance(clf.device_tokenizer, cabi.BPETokenizer)
    texts = bc.BPE_TRAPS + tc.random_texts(20, seed=3)
    if max_length == 8192:
        texts.append(" ".join(tc.random_texts(400, seed=5)))
    assert torch.equal(clf._embed_device(texts), clf._embed_ids_device(*clf._tokenize(texts)))
    labels = [f"c{i % 3}" for i in range(len(texts))]
    np.random.seed(0)
    clf.add_examples(texts, labels)
    q = tc.random_texts(24, seed=9) + ["a" * 5000]
    ids, mask, _ = clf._tokenize(q)
    assert clf.predict_batch(q, k=3) == clf.predict_batch_ids(ids, mask, k=3)
    clf.save(str(tmp_path / "saved"))
    loaded = acb.AdaptiveClassifier.load(str(tmp_path / "saved"), device="cuda")
    assert isinstance(loaded.device_tokenizer, cabi.BPETokenizer)
