"""Host tokenizer against the device WordPiece tokenizer, and predict_batch(texts) end to end with each
(profiles/h100_tokenize_bench.json).

Workload: seeded synthetic texts of ~110 words drawn from a seeded 30 k WordPiece vocab (some words capitalized, accented or
CJK), tokenized as AdaptiveClassifier does (max_length 128, truncation, padding).  Device and host outputs are checked equal
before anything is timed.  Times are host clocks around work that ends in a device synchronise.
    python tools/bench_tokenize.py [--out profiles/h100_tokenize_bench.json] [--reps 20]
"""
import argparse
import json
import os
import random
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402


def vocab_and_texts(n_texts: int, seed: int = 0):
    rng = random.Random(seed)
    letters = "abcdefghijklmnopqrstuvwxyz"
    specials = ["[PAD]", "[UNK]", "[CLS]", "[SEP]", "[MASK]"]
    vocab = specials + list(letters) + ["##" + c for c in letters] + list("éèüöçñ中文字国人大") + ["##" + c for c in "éèüöçñ"]
    seen = set(vocab)
    while len(vocab) < 30000:
        w = "".join(rng.choice(letters) for _ in range(rng.randint(2, 9)))
        w = w if rng.random() < 0.7 else "##" + w
        if w not in seen:
            seen.add(w)
            vocab.append(w)
    words = [w for w in vocab[5:] if not w.startswith("##")]
    texts = []
    for _ in range(n_texts):
        ws = []
        for _ in range(rng.randint(100, 120)):
            w = rng.choice(words)
            r = rng.random()
            if r < 0.1:
                w = w.capitalize()
            elif r < 0.15:
                w = w[:1] + "é" + w[1:]
            elif r < 0.18:
                w = "".join(rng.choice("中文字国人大") for _ in range(2))
            ws.append(w + ("," if rng.random() < 0.05 else ""))
        texts.append(" ".join(ws))
    return vocab, texts


def checkpoint(d: str, vocab, shape: str):
    from transformers import BertConfig, BertModel, BertTokenizerFast
    torch.manual_seed(0)
    dims = dict(minilm=(6, 384, 12, 1536), bert_base=(12, 768, 12, 3072))[shape]
    BertModel(BertConfig(vocab_size=len(vocab), num_hidden_layers=dims[0], hidden_size=dims[1], num_attention_heads=dims[2],
                         intermediate_size=dims[3])).eval().save_pretrained(d)
    BertTokenizerFast(vocab={w: i for i, w in enumerate(vocab)}, do_lower_case=True).save_pretrained(d)


def clock(fn, reps: int) -> float:
    fn()
    torch.cuda.synchronize()
    t = time.perf_counter()
    for _ in range(reps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_tokenize_bench.json"))
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs an H100"
    import subprocess
    import tokenizers
    import adaptive_classifier_b200 as acb
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()[0]
    res = dict(gpu=smi, cpus=len(os.sched_getaffinity(0)), tokenizers=tokenizers.__version__, max_length=128,
               words_per_text="100-120", tokenize={}, predict_batch={})
    vocab, texts = vocab_and_texts(512)
    with tempfile.TemporaryDirectory() as tmp:
        for shape in ("minilm", "bert_base"):
            d = os.path.join(tmp, shape)
            checkpoint(d, vocab, shape)
            clf = acb.AdaptiveClassifier(d, device="cuda", config={"max_length": 128})
            dev = clf.device_tokenizer
            assert dev is not None
            np.random.seed(0)
            clf.add_examples(texts[:40], [f"c{i % 4}" for i in range(40)])
            for B in (1, 32, 512):
                batch = texts[:B]
                ids, mask, tt = dev(batch, 128)
                hids, hmask, htt = clf._tokenize(batch)
                assert torch.equal(ids.cpu(), hids) and torch.equal(mask.cpu(), hmask) and torch.equal(tt.cpu(), htt)
                if shape == "minilm":
                    host = clock(lambda: clf._tokenize(batch), a.reps)
                    device = clock(lambda: dev(batch, 128), a.reps)
                    res["tokenize"][B] = dict(host_ms=host * 1e3, device_ms=device * 1e3, speedup=host / device)
                r = {}
                for path in ("host", "device"):
                    clf.device_tokenizer = dev if path == "device" else None
                    t = clock(lambda: clf.predict_batch(batch, k=3, batch_size=B), max(3, a.reps // 4))
                    r[f"{path}_texts_per_s"] = B / t
                clf.device_tokenizer = dev
                res["predict_batch"].setdefault(shape, {})[B] = r
                print(shape, B, res["tokenize"].get(B), r, flush=True)
    os.makedirs(os.path.dirname(a.out), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
