"""Seeded byte-level BPE tokenizers of the RoBERTa, ModernBERT and EuroBERT shapes, trained offline, and hand-made ones with
chosen merge lists, shared by the CPU (cpu_shim) and GPU tests of the device BPE tokenizer."""
import functools

import tokenizer_corpus as tc

LLAMA3 = (r"(?i:'s|'t|'re|'ve|'m|'ll|'d)|[^\r\n\p{L}\p{N}]?\p{L}+|\p{N}{1,3}| ?[^\s\p{L}\p{N}]+[\r\n]*|\s*[\r\n]+"
          r"|\s+(?!\S)|\s+")
KINDS = ["roberta", "roberta_prefix", "modernbert", "eurobert"]

# (content, normalized, lstrip, rstrip): every flag combination, and a normalized token that overlaps '<mask>'
FLAG_TOKENS = [(f"<t{n}{l}{r}>", bool(n), bool(l), bool(r)) for n in (0, 1) for l in (0, 1) for r in (0, 1)] + [
    ("b<m", True, False, False), ("zz", True, False, False), ("<t", False, False, False)]
SPACE_RUNS = [" " * n for n in range(24, 1, -1)]      # GPT-NeoX-style normalized added tokens for runs of spaces

BPE_TRAPS = tc.TRAPS + [
    "zab<mask>", "hi  \t<mask>", "q<mask>r", "<mask>", " <mask> ", "a <t011>  b<t001>\tc <t111> d", "<t010>x<t100> y <t110>\n",
    "x<t101>  y", "zzz zz<mask>zz", "b<mask>", "<t<t000>", "it's I'M they'RE we'Ve 'LL 'd 'ſ 'ß 'K", "don't", "'s's 's",
    "a1234567 12 ١٢٣٤ ½¾ x²", "\r\n\r\n x \n\n\ty\r", "a  \n  b", "   ", "\t\t", "  　 x y\u0085z", "$$$hello",
    "¿Qué? ¡Sí! «ok»", "  leading", "trailing  ", "tab\tend\t", "中文 字符abc123", "emoji 👩‍👩‍👧 ok", " a", "a ",
    " " * 30 + "x", "x" + " " * 25, "<|begin_of_text|> <|end_of_text|>", "<s></s><pad>", "[CLS] [MASK]x",
    "ｆｕｌｌ width", "x​y", "﻿bom", "é", "a'b 'c' ' '",
]


def _corpus(seed: int) -> list:
    return tc.random_texts(3000, seed=seed, words=(5, 60)) + BPE_TRAPS + [
        "the quick brown fox jumps over the lazy dog's back, isn't it? 12345 67 8.9"] * 50


def _wrap(tk, kind: str):
    from transformers import PreTrainedTokenizerFast
    if kind == "eurobert":
        return PreTrainedTokenizerFast(tokenizer_object=tk, bos_token="<|begin_of_text|>", eos_token="<|end_of_text|>",
                                       pad_token="<|end_of_text|>", model_input_names=["input_ids", "attention_mask"])
    if kind == "modernbert":
        return PreTrainedTokenizerFast(tokenizer_object=tk, cls_token="[CLS]", sep_token="[SEP]", pad_token="[PAD]",
                                       unk_token="[UNK]", mask_token="[MASK]", model_input_names=["input_ids", "attention_mask"])
    return PreTrainedTokenizerFast(tokenizer_object=tk, bos_token="<s>", eos_token="</s>", cls_token="<s>", sep_token="</s>",
                                   pad_token="<pad>", unk_token="<unk>", mask_token="<mask>",
                                   model_input_names=["input_ids", "attention_mask"])


def _finish(tk, kind: str, added: bool):
    """post-processor, special and added tokens of the kind, on a tokenizer whose model is set"""
    from tokenizers import AddedToken, pre_tokenizers, processors
    if kind == "eurobert":
        specials = ["<|begin_of_text|>", "<|end_of_text|>"] + [f"<|reserved_special_token_{i}|>" for i in range(6)]
        tk.add_special_tokens([AddedToken(s, normalized=False) for s in specials])
        bos, eos = tk.token_to_id(specials[0]), tk.token_to_id(specials[1])
        tk.post_processor = processors.TemplateProcessing(single=f"{specials[0]} $A {specials[1]}",
                                                          special_tokens=[(specials[0], bos), (specials[1], eos)])
    elif kind == "modernbert":
        tk.add_special_tokens([AddedToken("[MASK]", normalized=False, lstrip=True)] +
                              [AddedToken(s, normalized=False) for s in ("[UNK]", "[CLS]", "[SEP]", "[PAD]", "<|endoftext|>")])
        tk.add_tokens([AddedToken(s, normalized=True) for s in SPACE_RUNS])
        tk.post_processor = processors.Sequence([
            processors.ByteLevel(trim_offsets=False),
            processors.TemplateProcessing(single="[CLS] $A [SEP]", special_tokens=[("[CLS]", tk.token_to_id("[CLS]")),
                                                                                   ("[SEP]", tk.token_to_id("[SEP]"))])])
    else:
        tk.add_special_tokens([AddedToken(s, normalized=False) for s in ("<s>", "<pad>", "</s>", "<unk>")] +
                              [AddedToken("<mask>", normalized=False, lstrip=True)])
        tk.post_processor = processors.RobertaProcessing(("</s>", tk.token_to_id("</s>")), ("<s>", tk.token_to_id("<s>")))
    if added:
        for content, n, l, r in FLAG_TOKENS:
            if kind == "modernbert" and n and r:
                continue                 # next to the normalized space runs an rstrip token is refused
            tk.add_tokens([AddedToken(content, normalized=n, lstrip=l, rstrip=r, single_word=False)])
    return _wrap(tk, kind)


def _pre(kind: str):
    from tokenizers import Regex, pre_tokenizers
    if kind == "eurobert":
        return pre_tokenizers.Sequence([pre_tokenizers.Split(Regex(LLAMA3), "isolated"),
                                        pre_tokenizers.ByteLevel(add_prefix_space=False, use_regex=False)])
    return pre_tokenizers.ByteLevel(add_prefix_space=(kind == "roberta_prefix"))


@functools.lru_cache(maxsize=None)
def _trained(kind: str, vocab_size: int, seed: int):
    from tokenizers import Tokenizer, models, pre_tokenizers, trainers
    tk = Tokenizer(models.BPE(ignore_merges=(kind == "eurobert")))
    tk.pre_tokenizer = _pre(kind)
    # RoBERTa's specials lead its model vocab (the padding id is also its position embeddings' padding index)
    specials = ["<s>", "<pad>", "</s>", "<unk>", "<mask>"] if kind.startswith("roberta") else []
    tr = trainers.BpeTrainer(vocab_size=vocab_size, initial_alphabet=pre_tokenizers.ByteLevel.alphabet(), show_progress=False,
                             special_tokens=specials)
    tk.train_from_iterator(_corpus(seed), tr)
    return tk.to_str()


def make_bpe(kind: str, vocab_size: int = 4000, added: bool = True, seed: int = 0):
    """a tokenizer of `kind` (KINDS) trained on the seeded corpus to about vocab_size entries, wrapped as transformers does"""
    from tokenizers import Tokenizer
    return _finish(Tokenizer.from_str(_trained(kind, vocab_size, seed)), kind, added)


def make_handmade(kind: str, merges, extra=(), ignore_merges: bool = False, added: bool = False):
    """a tokenizer of `kind` whose model holds the 256 byte symbols, the tokens of `merges` (in that rank order) and `extra`"""
    from tokenizers import Tokenizer, models, pre_tokenizers
    vocab = {}
    for s in pre_tokenizers.ByteLevel.alphabet():
        vocab.setdefault(s, len(vocab))
    for a, b in merges:
        vocab.setdefault(a + b, len(vocab))
    for w in extra:
        vocab.setdefault(w, len(vocab))
    tk = Tokenizer(models.BPE(vocab=vocab, merges=list(merges), ignore_merges=ignore_merges))
    tk.pre_tokenizer = _pre(kind)
    return _finish(tk, kind, added)
