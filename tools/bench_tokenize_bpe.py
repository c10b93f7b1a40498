"""Host tokenizer against the device byte-level BPE tokenizer, and predict_batch(texts) end to end with each
(profiles/h100_tokenize_bpe_bench.json).

Workload: tools/bench_tokenize.py's seeded texts of 100-120 words, and byte-level BPE tokenizers trained to 30 k entries on
them, one with the GPT-2 split (RoBERTa / ModernBERT) and one with the Llama-3 split (EuroBERT).  Tokenized as
AdaptiveClassifier does (truncation, padding).  Device and host outputs are checked equal before anything is timed.  Also
timed in the same run: the WordPiece device tokenizer at B = 512, and one text made of a single word of AC_BPE_MAX_WORD bytes
(the longest word the device merges) on each path.  Times are host clocks around work that ends in a device synchronise.
    python tools/bench_tokenize_bpe.py [--out profiles/h100_tokenize_bpe_bench.json] [--reps 20]
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

import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench_tokenize import clock, vocab_and_texts  # noqa: E402

LLAMA3 = (r"(?i:'s|'t|'re|'ve|'m|'ll|'d)|[^\r\n\p{L}\p{N}]?\p{L}+|\p{N}{1,3}| ?[^\s\p{L}\p{N}]+[\r\n]*|\s*[\r\n]+"
          r"|\s+(?!\S)|\s+")


def bpe_tokenizer(texts, split: str):
    """a 30 k byte-level BPE trained on the texts: 'gpt2' with RobertaProcessing (RoBERTa's shape), 'llama3' with the
    Llama-3 split, ignore_merges and '<|begin_of_text|> $A <|end_of_text|>' (EuroBERT's)"""
    from tokenizers import AddedToken, Regex, Tokenizer, models, pre_tokenizers, processors, trainers
    from transformers import PreTrainedTokenizerFast
    tk = Tokenizer(models.BPE(ignore_merges=(split == "llama3")))
    if split == "llama3":
        tk.pre_tokenizer = pre_tokenizers.Sequence([pre_tokenizers.Split(Regex(LLAMA3), "isolated"),
                                                    pre_tokenizers.ByteLevel(add_prefix_space=False, use_regex=False)])
        specials = ["<|begin_of_text|>", "<|end_of_text|>"]
    else:
        tk.pre_tokenizer = pre_tokenizers.ByteLevel(add_prefix_space=False)
        specials = ["<s>", "<pad>", "</s>", "<unk>", "<mask>"]
    tk.train_from_iterator(texts, trainers.BpeTrainer(vocab_size=30000, show_progress=False,      # RoBERTa's specials lead its vocab
                                                      special_tokens=specials if split == "gpt2" else [],
                                                      initial_alphabet=pre_tokenizers.ByteLevel.alphabet()))
    tk.add_special_tokens([AddedToken(s, normalized=False, lstrip=(s == "<mask>")) for s in specials])
    if split == "llama3":
        bos, eos = (tk.token_to_id(s) for s in specials)
        tk.post_processor = processors.TemplateProcessing(single=f"{specials[0]} $A {specials[1]}",
                                                          special_tokens=[(specials[0], bos), (specials[1], eos)])
        return PreTrainedTokenizerFast(tokenizer_object=tk, bos_token=specials[0], eos_token=specials[1],
                                       pad_token=specials[1], model_input_names=["input_ids", "attention_mask"])
    tk.post_processor = processors.RobertaProcessing(("</s>", tk.token_to_id("</s>")), ("<s>", tk.token_to_id("<s>")))
    return PreTrainedTokenizerFast(tokenizer_object=tk, bos_token="<s>", eos_token="</s>", cls_token="<s>", sep_token="</s>",
                                   pad_token="<pad>", unk_token="<unk>", mask_token="<mask>",
                                   model_input_names=["input_ids", "attention_mask"])


def checkpoint(d: str, tok, shape: str):
    from transformers import ModernBertConfig, ModernBertModel, RobertaConfig, RobertaModel
    torch.manual_seed(0)
    if shape == "roberta_base":
        m = RobertaModel(RobertaConfig(vocab_size=len(tok), hidden_size=768, num_hidden_layers=12, num_attention_heads=12,
                                       intermediate_size=3072, max_position_embeddings=514, pad_token_id=tok.pad_token_id))
    else:
        m = ModernBertModel(ModernBertConfig(vocab_size=len(tok), hidden_size=768, num_hidden_layers=22, num_attention_heads=12,
                                             intermediate_size=1152, max_position_embeddings=8192,
                                             pad_token_id=tok.pad_token_id, cls_token_id=tok.cls_token_id,
                                             sep_token_id=tok.sep_token_id, bos_token_id=tok.cls_token_id,
                                             eos_token_id=tok.sep_token_id))
    m.eval().save_pretrained(d)
    tok.save_pretrained(d)


def check_equal(dev, tok, batch, max_length):
    ids, mask, _ = dev(batch, max_length)
    ref = tok(batch, max_length=max_length, truncation=True, padding=True, return_tensors="pt")
    assert torch.equal(ids.cpu(), ref["input_ids"].to(torch.int32)) and torch.equal(mask.cpu(), ref["attention_mask"].to(torch.int32))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_tokenize_bpe_bench.json"))
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs an H100"
    import tokenizers
    import adaptive_classifier_b200 as acb
    from adaptive_classifier_b200 import _cabi
    from adaptive_classifier_b200.tokenizer import MAX_WORD
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()[0]
    res = dict(gpu=smi, cpus=len(os.sched_getaffinity(0)), tokenizers=tokenizers.__version__, words_per_text="100-120",
               tokenize={}, long_word={}, wordpiece_b512={}, predict_batch={})
    vocab, texts = vocab_and_texts(512)
    long_texts = [" ".join(texts[8 * i: 8 * i + 8]) * 2 for i in range(8)]         # ~1,800 words each: past 8192 tokens
    toks = {}
    for split in ("gpt2", "llama3"):
        tok = bpe_tokenizer(texts, split)
        toks[split] = tok
        dev, why = _cabi.BPETokenizer.from_hf(tok)
        assert dev is not None, why
        r = res["tokenize"][split] = {}
        for B, max_length, batch in ((1, 128, texts[:1]), (32, 128, texts[:32]), (512, 128, texts), (8, 8192, long_texts)):
            check_equal(dev, tok, batch, max_length)
            host = clock(lambda: tok(batch, max_length=max_length, truncation=True, padding=True, return_tensors="pt"), a.reps)
            device = clock(lambda: dev(batch, max_length), a.reps)
            r[f"B{B}_L{max_length}"] = dict(host_ms=host * 1e3, device_ms=device * 1e3, speedup=host / device)
            print(split, B, max_length, r[f"B{B}_L{max_length}"], flush=True)
        word = ["".join(np.random.default_rng(0).choice(list("abcdefghijklmnopqrstuvwxyz"), MAX_WORD))]
        check_equal(dev, tok, word, 128)
        res["long_word"][split] = dict(bytes=MAX_WORD, host_ms=clock(lambda: tok(word, max_length=128, truncation=True), a.reps) * 1e3,
                                       device_ms=clock(lambda: dev(word, 128), a.reps) * 1e3)
        print(split, "word", res["long_word"][split], flush=True)
    with tempfile.TemporaryDirectory() as tmp:
        wp = os.path.join(tmp, "wp")
        from bench_tokenize import checkpoint as wp_checkpoint
        wp_checkpoint(wp, vocab, "minilm")
        clf = acb.AdaptiveClassifier(wp, device="cuda", config={"max_length": 128})
        assert isinstance(clf.device_tokenizer, _cabi.WordPieceTokenizer)
        dev = clf.device_tokenizer
        res["wordpiece_b512"] = dict(host_ms=clock(lambda: clf._tokenize(texts), a.reps) * 1e3,
                                     device_ms=clock(lambda: dev(texts, 128), a.reps) * 1e3)
        print("wordpiece", res["wordpiece_b512"], flush=True)
        del clf
        for shape in ("roberta_base", "modernbert_base"):
            d = os.path.join(tmp, shape)
            checkpoint(d, toks["gpt2"], shape)
            clf = acb.AdaptiveClassifier(d, device="cuda", config={"max_length": 128})
            dev = clf.device_tokenizer
            assert isinstance(dev, _cabi.BPETokenizer)
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
