"""Device WordPiece tokenizer on the H100: the kernel's ids against the Hugging Face tokenizer call, and the classifier's text
path through it against the host-tokenized path, bit for bit."""
import numpy as np
import pytest
import torch

import tokenizer_corpus as tc

pytestmark = pytest.mark.gpu

KINDS = ["bert", "bert_cased", "electra", "mpnet"]


def _batch(B: int, max_length: int) -> list:
    texts = tc.TRAPS + tc.random_texts(64, seed=B + max_length) + ["a" * 1_000_000]
    if max_length == 8192:
        texts.append(" ".join(tc.random_texts(400, seed=5)))           # past 8192 tokens: truncated
    return (texts * (B // len(texts) + 1))[:B] if B > len(texts) else texts[-B:] if B < 8 else texts[:B]


@pytest.mark.parametrize("kind", KINDS)
def test_device_ids_equal_hf(cabi, kind):
    tok = tc.make_tokenizer(kind)
    dev, why = cabi.WordPieceTokenizer.from_hf(tok)
    assert dev is not None, why
    for max_length in (8, 128, 512, 8192):
        for B in (1, 7, 512, 1024):
            texts = _batch(B, max_length)
            ids, mask, tt = dev(texts, max_length)
            torch.cuda.synchronize()
            ref = tok(texts, max_length=max_length, truncation=True, padding=True, return_tensors="pt")
            assert torch.equal(ids.cpu(), ref["input_ids"].to(torch.int32)), (kind, max_length, B)
            assert torch.equal(mask.cpu(), ref["attention_mask"].to(torch.int32))
            if "token_type_ids" in ref:
                assert torch.equal(tt.cpu(), ref["token_type_ids"].to(torch.int32))
            else:
                assert tt is None
    assert dev(["ok", "bad \ud800 surrogate"], 16) is None                 # no UTF-8 form: the caller's host path decides


def _checkpoint(tmp_path, kind: str) -> str:
    from transformers import (BertConfig, BertModel, MPNetConfig, MPNetModel, RobertaConfig, RobertaModel,
                              RobertaTokenizer)
    torch.manual_seed(11)
    d = str(tmp_path / kind)
    if kind == "roberta":
        vocab = {w: i for i, w in enumerate(["<s>", "<pad>", "</s>", "<unk>", "<mask>"] + list("abcdefghij") + ["Ġ" + c for c in "abcdefghij"])}
        tok = RobertaTokenizer(vocab=vocab, merges=[])
        m = RobertaModel(RobertaConfig(vocab_size=len(vocab), hidden_size=128, num_hidden_layers=2, num_attention_heads=2,
                                       intermediate_size=256, max_position_embeddings=130, pad_token_id=1))
    else:
        tok = tc.make_tokenizer(kind)
        cfg = dict(vocab_size=len(tok), hidden_size=128, num_hidden_layers=2, num_attention_heads=2, intermediate_size=256)
        m = MPNetModel(MPNetConfig(**cfg)) if kind == "mpnet" else BertModel(BertConfig(**cfg))
    m.eval().save_pretrained(d)
    tok.save_pretrained(d)
    return d


@pytest.mark.parametrize("kind", ["bert", "mpnet"])
def test_classifier_text_path_is_bitwise_the_host_path(cabi, tmp_path, kind):
    import adaptive_classifier_b200 as acb
    clf = acb.AdaptiveClassifier(_checkpoint(tmp_path, kind), device="cuda")
    assert clf.device_tokenizer is not None
    texts = tc.TRAPS + tc.random_texts(20, seed=3)
    assert torch.equal(clf._embed_device(texts), clf._embed_ids_device(*clf._tokenize(texts)))
    labels = [f"c{i % 3}" for i in range(len(texts))]
    np.random.seed(0)
    clf.add_examples(texts, labels)
    q = tc.random_texts(24, seed=9)
    ids, mask, _ = clf._tokenize(q)
    assert clf.predict_batch(q, k=3) == clf.predict_batch_ids(ids, mask, k=3)
    clf.save(str(tmp_path / "saved"))
    assert acb.AdaptiveClassifier.load(str(tmp_path / "saved"), device="cuda").device_tokenizer is not None


def test_roberta_tokenizer_stays_on_the_host(cabi, tmp_path):
    import adaptive_classifier_b200 as acb
    clf = acb.AdaptiveClassifier(_checkpoint(tmp_path, "roberta"), device="cuda")
    assert clf.device_tokenizer is None
    texts = ["abc def", "ghij", "a b c d e f"]
    assert torch.equal(clf._embed_device(texts), clf._embed_ids_device(*clf._tokenize(texts)))


def test_classifier_keeps_the_host_path_when_the_device_tokenizer_cannot_be_built(cabi, tmp_path, monkeypatch):
    """a WordPiece vocab with an empty entry (a blank line in vocab.txt) is refused by wordpiece_spec, and a failure while
    building the handle is logged: either way the classifier is constructed and tokenizes on the host"""
    from transformers import BertConfig, BertModel, BertTokenizerFast
    import adaptive_classifier_b200 as acb
    d = str(tmp_path / "blank")
    vocab = tc.SPECIALS_BERT + ["", "abc", "def"]
    BertModel(BertConfig(vocab_size=len(vocab), hidden_size=128, num_hidden_layers=2, num_attention_heads=2,
                         intermediate_size=256)).eval().save_pretrained(d)
    BertTokenizerFast(vocab={w: i for i, w in enumerate(vocab)}).save_pretrained(d)
    clf = acb.AdaptiveClassifier(d, device="cuda")
    assert clf.device_tokenizer is None
    texts = ["abc def", "def xyz abc"]
    assert torch.equal(clf._embed_device(texts), clf._embed_ids_device(*clf._tokenize(texts)))

    def fail(self, spec, device="cuda"):
        raise cabi.AdaptiveB200Error("ac_tokenizer_create failed (rc=-2): out of memory")
    monkeypatch.setattr(cabi.WordPieceTokenizer, "__init__", fail)
    clf = acb.AdaptiveClassifier(_checkpoint(tmp_path, "bert"), device="cuda")
    assert clf.device_tokenizer is None
    assert torch.equal(clf._embed_device(texts), clf._embed_ids_device(*clf._tokenize(texts)))
