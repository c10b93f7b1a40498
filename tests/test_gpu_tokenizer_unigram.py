"""Device SentencePiece Unigram tokenizer on the H100: the kernels' ids against the Hugging Face tokenizer call for XLM-R-shaped
tokenizers of each built-in normalization rule, and the classifier's text path through it against the host-tokenized path,
bit for bit, on a seeded XLM-R-shaped local checkpoint."""
import numpy as np
import pytest
import torch

import unigram_corpus as uc

pytestmark = pytest.mark.gpu


def _batch(B: int, max_length: int) -> list:
    texts = uc.UNIGRAM_TRAPS + uc.random_texts(64, seed=B + max_length) + ["a" * 1_000_000, "x " + "日" * 300_000 + " y"]
    if max_length == 8192:
        texts.append(" ".join(uc.random_texts(400, seed=5)))           # past 8192 tokens: truncated
    return (texts * (B // len(texts) + 1))[:B] if B > len(texts) else texts[-B:] if B < 8 else texts[:B]


@pytest.mark.parametrize("rule,vocab_size", [("nmt_nfkc", 8000), ("nmt_nfkc", 30000), ("nfkc", 8000), ("nmt_nfkc_cf", 8000)])
def test_device_ids_equal_hf(cabi, rule, vocab_size):
    tok = uc.make_unigram(rule, vocab_size)
    dev, why = cabi.UnigramTokenizer.from_hf(tok)
    assert dev is not None, why
    for max_length in (8, 128, 512, 8192):
        for B in (1, 7, 512, 1024):
            texts = _batch(B, max_length)
            ids, mask, tt = dev(texts, max_length)
            torch.cuda.synchronize()
            ref = tok(texts, max_length=max_length, truncation=True, padding=True, return_tensors="pt")
            assert torch.equal(ids.cpu(), ref["input_ids"].to(torch.int32)), (rule, max_length, B)
            assert torch.equal(mask.cpu(), ref["attention_mask"].to(torch.int32))
            assert tt is None and "token_type_ids" not in ref
    assert dev(["ok", "bad \ud800 surrogate"], 16) is None                 # no UTF-8 form: the caller's host path decides


def test_handmade_lattices_on_the_device(cabi):
    """score ties, fused unknown chars, the special pieces as text and '▁', as the CPU shim runs them"""
    tok = uc.make_handmade([("▁", -1.0), ("a", -2.0), ("b", -2.0), ("ab", -4.0), ("▁ab", -5.0), ("▁a", -3.0), ("x", -9.0),
                            ("y", -9.0), ("xy", -18.0), ("▁x", -9.0)])
    texts = ["ab", "abab", "xyxy", "zzz", "qzq", "a qqq b", "▁ab", "a▁▁b", "<s>ab</s>", "x <mask>", "<unk>", "q<s>q"]
    dev, why = cabi.UnigramTokenizer.from_hf(tok)
    assert dev is not None, why
    ids, mask, _ = dev(texts, 32)
    ref = tok(texts, max_length=32, truncation=True, padding=True, return_tensors="pt")
    assert torch.equal(ids.cpu(), ref["input_ids"].to(torch.int32)) and torch.equal(mask.cpu(), ref["attention_mask"].to(torch.int32))


def _checkpoint(tmp_path) -> str:
    from transformers import XLMRobertaConfig, XLMRobertaModel
    torch.manual_seed(11)
    d = str(tmp_path / "xlmr")
    import os
    os.makedirs(d)
    n = uc.save_pretrained_tokenizer(d)
    m = XLMRobertaModel(XLMRobertaConfig(vocab_size=n, hidden_size=128, num_hidden_layers=2, num_attention_heads=2,
                                         intermediate_size=256, max_position_embeddings=8194, pad_token_id=1,
                                         bos_token_id=0, eos_token_id=2))
    m.eval().save_pretrained(d)
    return d


@pytest.mark.parametrize("max_length", [512, 8192])
def test_classifier_text_path_is_bitwise_the_host_path(cabi, tmp_path, max_length):
    import adaptive_classifier_b200 as acb
    config = {"max_length": max_length} if max_length != 512 else {}
    clf = acb.AdaptiveClassifier(_checkpoint(tmp_path), device="cuda", config=config)
    assert isinstance(clf.device_tokenizer, cabi.UnigramTokenizer)
    texts = uc.UNIGRAM_TRAPS[:-6] + uc.random_texts(20, seed=3)
    if max_length == 8192:
        texts.append(" ".join(uc.random_texts(400, seed=5)))
    assert torch.equal(clf._embed_device(texts), clf._embed_ids_device(*clf._tokenize(texts)))
    labels = [f"c{i % 3}" for i in range(len(texts))]
    np.random.seed(0)
    clf.add_examples(texts, labels)
    q = uc.random_texts(24, seed=9) + ["日" * 5000]
    ids, mask, _ = clf._tokenize(q)
    assert clf.predict_batch(q, k=3) == clf.predict_batch_ids(ids, mask, k=3)
    clf.save(str(tmp_path / "saved"))
    loaded = acb.AdaptiveClassifier.load(str(tmp_path / "saved"), device="cuda")
    assert isinstance(loaded.device_tokenizer, cabi.UnigramTokenizer)
