#!/usr/bin/env python
"""Bitwise comparison of two builds of libadaptive_b200.so on the encoder attention variants.

    python tools/compare_attention_builds.py --other /path/to/the/other/libadaptive_b200.so

For a change that is meant to leave the attention arithmetic and its order alone, "within tolerance" is too weak: this runs
the same seeded inputs through this tree's library and through `--other` (say, the parent commit built elsewhere), each in
a process of its own, and compares the outputs with torch.equal.  One encoder per attention variant, two layers each
(ModernBERT three: one full, two sliding), three sequences of lengths S, S - 37 and min(S, 90) under a padding mask:

    BERT-base shape (head_dim 64)   S 128, 384      MPNet       S 128, 384      ModernBERT (half-window 64)   S 1024
    MiniLM shape (head_dim 32)      S 128, 384      DeBERTa-v3  S 77, 384       EuroBERT (RMSNorm, SwiGLU)    S 128, 384
    ALBERT (E = 128, tanh GELU)     S 128, 384      NomicBERT (post-LN RoPE, SwiGLU)  S 128, 384

so that every layer-loop instantiation (post-LN with erf / tanh GELU, with RoPE and SwiGLU, the embedding projection;
pre-LN with LayerNorm / GeGLU and RMSNorm / SwiGLU) runs.

Per case: `Encoder.forward_cls` (unit CLS rows, fp32) and `Encoder.attention` on seeded q, k, v (the stage alone, fp16; with
the sliding half-window on ModernBERT).  Prints one line per case and exits 1 if any bit differs.  Writes only to a
temporary directory.

A library that sits in a built source tree (next to its own _cabi.py, as adaptive_classifier_b200/libadaptive_b200.so
does) is driven by that tree's bindings, so builds whose C ABI or table layouts differ are each called as their own
Python calls them.
"""
import argparse
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

VOCAB = 2000
CASES = (("bert", (128, 384)), ("minilm", (128, 384)), ("mpnet", (128, 384)), ("deberta", (77, 384)), ("modernbert", (1024,)),
         ("eurobert", (128, 384)), ("albert", (128, 384)), ("nomic", (128, 384)))


def model(name):
    import transformers as tf
    torch.manual_seed(1234)
    if name in ("bert", "minilm"):
        dims = {"bert": dict(hidden_size=768, intermediate_size=3072), "minilm": dict(hidden_size=384, intermediate_size=1536)}
        cfg = tf.BertConfig(vocab_size=VOCAB, num_hidden_layers=2, num_attention_heads=12, **dims[name])
        return tf.BertModel(cfg, add_pooling_layer=False).eval()
    if name == "mpnet":
        cfg = tf.MPNetConfig(vocab_size=VOCAB, hidden_size=768, num_hidden_layers=2, num_attention_heads=12,
                             intermediate_size=3072, max_position_embeddings=514, layer_norm_eps=1e-5)
        return tf.MPNetModel(cfg, add_pooling_layer=False).eval()
    if name == "deberta":
        cfg = tf.DebertaV2Config(vocab_size=VOCAB, hidden_size=768, num_hidden_layers=2, num_attention_heads=12,
                                 intermediate_size=3072, max_position_embeddings=512, type_vocab_size=0,
                                 relative_attention=True, position_buckets=256, norm_rel_ebd="layer_norm", share_att_key=True,
                                 pos_att_type=["p2c", "c2p"], position_biased_input=False, layer_norm_eps=1e-7,
                                 hidden_act="gelu", pad_token_id=0)
        m = tf.DebertaV2Model(cfg).eval()
        with torch.no_grad():          # N(0, 1) relative embeddings, so that the position terms move the scores
            m.encoder.rel_embeddings.weight.normal_(0.0, 1.0)
        return m
    if name == "eurobert":
        cfg = tf.EuroBertConfig(vocab_size=VOCAB, hidden_size=768, num_hidden_layers=2, num_attention_heads=12,
                                num_key_value_heads=4, intermediate_size=2048, max_position_embeddings=8192, bos_token_id=0,
                                eos_token_id=2, pad_token_id=1, mask_token_id=3)
        return tf.EuroBertModel(cfg).eval()
    if name == "albert":
        cfg = tf.AlbertConfig(vocab_size=VOCAB, embedding_size=128, hidden_size=768, num_hidden_layers=2,
                              num_attention_heads=12, intermediate_size=3072, hidden_act="gelu_new")
        return tf.AlbertModel(cfg, add_pooling_layer=False).eval()
    if name == "nomic":
        cfg = tf.NomicBertConfig(vocab_size=VOCAB, hidden_size=768, num_hidden_layers=2, num_attention_heads=12,
                                 intermediate_size=3072, max_position_embeddings=2048, type_vocab_size=2)
        return tf.NomicBertModel(cfg).eval()
    cfg = tf.ModernBertConfig(vocab_size=VOCAB, num_hidden_layers=3, pad_token_id=VOCAB - 1, bos_token_id=VOCAB - 3,
                              eos_token_id=VOCAB - 2, cls_token_id=VOCAB - 3, sep_token_id=VOCAB - 2)
    return tf.ModernBertModel(cfg).eval()


def emit(lib, out_path):
    pkg = os.path.dirname(os.path.abspath(lib))
    if os.path.exists(os.path.join(pkg, "_cabi.py")):
        sys.path.insert(0, os.path.dirname(pkg))
    from adaptive_classifier_b200 import _cabi
    _cabi.LIB_PATH = lib
    _cabi.load_library()
    dev = torch.device("cuda", 0)
    out = {}
    for name, seqs in CASES:
        enc = _cabi.Encoder.from_hf(model(name), max_tokens=3 * max(seqs), device=dev)
        dh = enc.hidden // enc.heads
        for S in seqs:
            g = torch.Generator().manual_seed(100 + S)
            lens = torch.tensor([S, S - 37, min(S, 90)])
            mask = (torch.arange(S)[None, :] < lens[:, None]).to(torch.int32).to(dev)
            ids = torch.randint(10, VOCAB - 10, (3, S), generator=g, dtype=torch.int64).to(torch.int32).to(dev)
            out[f"{name} S={S} forward_cls"] = enc.forward_cls(ids, mask).cpu()
            q, k, v = (torch.randn(3, S, enc.heads, dh, generator=g).to(dev) for _ in range(3))
            window = 64 if name == "modernbert" else 0
            out[f"{name} S={S} attention"] = enc.attention(2.0 * q, 2.0 * k, v, mask, window=window).cpu()
        enc.close()
    torch.save(out, out_path)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--other", help="the other build's libadaptive_b200.so")
    ap.add_argument("--emit", nargs=2, metavar=("LIB", "OUT"), help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.emit:
        return emit(*args.emit)
    if not args.other or not os.path.exists(args.other):
        ap.error("--other must name an existing library")
    if not torch.cuda.is_available():
        raise SystemExit("compare_attention_builds.py: no CUDA device; the CUDA path has no CPU fallback")
    from adaptive_classifier_b200 import _cabi
    with tempfile.TemporaryDirectory() as tmp:
        outs = []
        for i, lib in enumerate((_cabi.LIB_PATH, os.path.abspath(args.other))):
            path = os.path.join(tmp, f"{i}.pt")
            subprocess.check_call([sys.executable, os.path.abspath(__file__), "--emit", lib, path])
            outs.append(torch.load(path))
    differing = 0
    for key, a in outs[0].items():
        b = outs[1][key]
        same = a.dtype == b.dtype and a.shape == b.shape and torch.equal(a, b)
        sane = bool(torch.isfinite(a.float()).all()) and float(a.float().abs().max()) > 0.0
        differing += not (same and sane)
        note = "" if same else f"  max |a - b| {float((a.float() - b.float()).abs().max()):.3e}"
        print(f"{key:36s} {'equal' if same else 'DIFFERENT'}{'' if sane else '  (not finite or all zero)'}{note}")
    print(f"{len(outs[0])} outputs, {differing} differing")
    sys.exit(1 if differing else 0)


if __name__ == "__main__":
    main()
