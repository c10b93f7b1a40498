"""Host tokenizer against the device SentencePiece Unigram tokenizer (XLM-RoBERTa shape), and predict_batch(texts) end to end
with each (profiles/h100_tokenize_unigram_bench.json).

Workload: the seeded mixed-script texts of tests/unigram_corpus.py (Latin with accents, Cyrillic, Arabic, Devanagari, CJK and
kana runs that WhitespaceSplit leaves as long words, fullwidth forms, ligatures, emoji), and a Unigram model sentencepiece
trains to 30 k pieces on them with its nmt_nfkc rule (XLM-R's), loaded through AutoTokenizer as an XLM-R tokenizer.
Tokenized as AdaptiveClassifier does (truncation, padding).  Device and host outputs are checked equal before anything is
timed.  Also timed: one text made of a single word of 512 to AC_UNIGRAM_MAX_WORD bytes on each path (Latin and CJK), which
places the bound above which a word is left to the host.  predict_batch runs on random-weight encoders of the
xlm-roberta-large / bge-m3 shape and the multilingual-e5-base shape with this 30 k vocab.  Times are host clocks around work
that ends in a device synchronise.
    python tools/bench_tokenize_unigram.py [--out profiles/h100_tokenize_unigram_bench.json] [--reps 20]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench_tokenize import clock  # noqa: E402
import unigram_corpus as uc  # noqa: E402


def checkpoint(d: str, shape: str) -> None:
    from transformers import XLMRobertaConfig, XLMRobertaModel
    os.makedirs(d)
    n = uc.save_pretrained_tokenizer(d, vocab_size=30000)
    torch.manual_seed(0)
    if shape == "xlmr_large":          # xlm-roberta-large / bge-m3 / arctic-embed-l-v2.0
        cfg = dict(hidden_size=1024, num_hidden_layers=24, num_attention_heads=16, intermediate_size=4096,
                   max_position_embeddings=8194)
    else:                              # multilingual-e5-base
        cfg = dict(hidden_size=768, num_hidden_layers=12, num_attention_heads=12, intermediate_size=3072,
                   max_position_embeddings=514)
    XLMRobertaModel(XLMRobertaConfig(vocab_size=n, pad_token_id=1, bos_token_id=0, eos_token_id=2, **cfg)).eval().save_pretrained(d)


def check_equal(dev, tok, batch, max_length):
    ids, mask, _ = dev(batch, max_length)
    ref = tok(batch, max_length=max_length, truncation=True, padding=True, return_tensors="pt")
    assert torch.equal(ids.cpu(), ref["input_ids"].to(torch.int32)) and torch.equal(mask.cpu(), ref["attention_mask"].to(torch.int32))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_tokenize_unigram_bench.json"))
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs an H100"
    import tokenizers
    import adaptive_classifier_b200 as acb
    from adaptive_classifier_b200 import _cabi
    from adaptive_classifier_b200.tokenizer import UNIGRAM_MAX_WORD
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()[0]
    res = dict(gpu=smi, cpus=len(os.sched_getaffinity(0)), tokenizers=tokenizers.__version__, words_per_text="60-80",
               tokenize={}, long_word={}, predict_batch={})
    texts = uc.random_texts(512, seed=1, words=(60, 80))
    long_texts = [" ".join(texts[8 * i: 8 * i + 8]) * 3 for i in range(8)]
    tok = uc.make_unigram("nmt_nfkc", 30000)
    dev, why = _cabi.UnigramTokenizer.from_hf(tok)
    assert dev is not None, why
    res["text_bytes_b512"] = sum(len(t.encode()) for t in texts)
    for B, max_length, batch in ((1, 128, texts[:1]), (32, 128, texts[:32]), (512, 128, texts), (8, 8192, long_texts)):
        check_equal(dev, tok, batch, max_length)
        host = clock(lambda: tok(batch, max_length=max_length, truncation=True, padding=True, return_tensors="pt"), a.reps)
        device = clock(lambda: dev(batch, max_length), a.reps)
        res["tokenize"][f"B{B}_L{max_length}"] = dict(host_ms=host * 1e3, device_ms=device * 1e3, speedup=host / device)
        print(B, max_length, res["tokenize"][f"B{B}_L{max_length}"], flush=True)
    rng = np.random.default_rng(0)
    for script, alpha in (("latin", list("abcdefghijklmnopqrstuvwxyz")), ("cjk", list(uc.SCRIPTS["cjk"]))):
        for nbytes in (512, 1024, 2048, UNIGRAM_MAX_WORD):
            per = len(alpha[0].encode())
            word = ["".join(rng.choice(alpha, (nbytes - 3) // per))]
            check_equal(dev, tok, word, 128)
            r = dict(host_ms=clock(lambda: tok(word, max_length=128, truncation=True, padding=True, return_tensors="pt"),
                                   a.reps) * 1e3,
                     device_ms=clock(lambda: dev(word, 128), a.reps) * 1e3)
            res["long_word"][f"{script}_{nbytes}"] = r
            print("word", script, nbytes, r, flush=True)
    with tempfile.TemporaryDirectory() as tmp:
        for shape in ("xlmr_large", "me5_base"):
            d = os.path.join(tmp, shape)
            checkpoint(d, shape)
            clf = acb.AdaptiveClassifier(d, device="cuda", config={"max_length": 128})
            dev = clf.device_tokenizer
            assert isinstance(dev, _cabi.UnigramTokenizer)
            np.random.seed(0)
            clf.add_examples(texts[:40], [f"c{i % 4}" for i in range(40)])
            for B in (1, 32, 512):
                batch = texts[:B]
                r = {}
                for path in ("host", "device"):
                    clf.device_tokenizer = dev if path == "device" else None
                    t = clock(lambda: clf.predict_batch(batch, k=3, batch_size=B), max(3, a.reps // 4))
                    r[f"{path}_texts_per_s"] = B / t
                clf.device_tokenizer = dev
                res["predict_batch"].setdefault(shape, {})[B] = r
                print(shape, B, r, flush=True)
            del clf
    os.makedirs(os.path.dirname(a.out), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
