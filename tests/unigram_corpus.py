"""Seeded SentencePiece Unigram tokenizers of the XLM-RoBERTa shape, trained offline by sentencepiece on a multilingual corpus
with its built-in normalization rules and loaded through AutoTokenizer (so the pipeline transformers builds is what runs),
and hand-built ones with chosen pieces and scores, shared by the CPU (cpu_shim) and GPU tests of the device Unigram
tokenizer."""
import functools
import io
import json
import os
import random
import tempfile

RULES = ["nmt_nfkc", "nfkc", "nmt_nfkc_cf"]
# per script: letters the random words are drawn from
SCRIPTS = {
    "latin": "abcdefghijklmnopqrstuvwxyzéèêëàâäôöûüçñßøåæœ",
    "caps": "ABCDEFGHIJKLMNOPQRSTUVWXYZÉÀÖÜÑ",
    "cyrillic": "абвгдеёжзийклмнопрстуфхцчшщъыьэюя",
    "arabic": "ابتثجحخدذرزسشصضطظعغفقكلمنهوي",
    "devanagari": "कखगघचछजझटठडढणतथदधनपफबभमयरलवशषसह" + "ािीुूेैोौं्",
    "cjk": "的一是不了人我在有他这中大来上国个到说们为子和你地出道也时年得就那要下以生会自着去之过家学对可她里后小么心多天而能好都然没日于起还发成事只作当想看文无开手十用主行方又如前所本见经头面公同三已老从动两长知民样现分将外但身些与高意进把法此实回二理美点月明其种声全工己话儿者向情部正名定女问力机给等几很业最间新什打便位因重被走电四第门相次东政海口使教西再平真听世气信北少关并内加化由却代军产入先山五太水万市眼体别处总才场师书比住员九笑性通目华报立马命张活难神数件安表原车白应路期叫死常提感金何更反合放做系计或司利受光王果亲界及今京务制解各任至清物台象记边共风战干接它许八特觉望直服毛林题建南度统色字请交爱让认算论百吃义科怎元社术结六功指思非流每青管夫连远资队跟带花快条院变联言权往展该由",
    "hiragana": "あいうえおかきくけこさしすせそたちつてとなにぬねのはひふへほまみむめもやゆよらりるれろわをんがぎぐげござじずぜぞだでどばびぶべぼぱぴぷぺぽ",
    "fullwidth": "ＡＢＣＤＥＦＧｆｕｌｌｗｉｄｔｈ０１２３４５",
    "ligature": "ﬁﬂﬀﬃﬄ",
}
EXTRAS = ["①", "②", "㎏", "™", "½", "Ⅻ", "ǅ", "ﷺ", "👍", "😀", "👩‍👩‍👧", "🇫🇷", "中文", "日本語", "한국어", "Á", "ë́",
          "क्ष", "x​y", "a　b", "\r\n", "\t", "İ", "ς", "Å", "ﬀ"]
# the library behaviours the device kernels reproduce, in texts: Precompiled on clusters, whitespace of every kind, added
# tokens next to and inside words, the special pieces as plain text, the metaspace char itself
UNIGRAM_TRAPS = [
    "Ａ́ ①́ ｆ́x ｆ̈́ ｆ‍ ｆि", "\r\n x\r\ny x​x a　b", "Hello World", "  déjà vu, NAÏVE café!  ", "中文字符 and 𠀀",
    "İstanbul ΣΟΦΟΣ", "a\tb\nc d　e", "tab\x00null�", "emoji 👩‍👩‍👧 $5+<3>", "x" * 120, "▁", "a▁▁b", "▁▁a a▁", "a ▁ b",
    "<s> </s> <pad> <unk> <mask>", "x<mask>y <mask>", "hi  \t<mask>", "<s><s>x</s>", "▁<s>▁", "xyz 🤖🤖 qqq", "ﷺ ﷺﷺ",
    "ｆｕｌｌ ｗｉｄｔｈ ＡＢＣ", "ﬁle ﬂow ǅ Ⅻ ㎏ ½", "नमस्ते क्षत्रिय", "مرحبا بالعالم", "привет мир", "日本語のテキスト",
    "ẹ̈́ Å", "؀x ؀؀y", "á́́́", "각", "🇫🇷🇩🇪",
    "b\u0307 ab\u0307c abb\u0323a b\u0307 B\u0307\u0323 d\u0307",      # decomposed: keys of two and three chars
    "", " ", "   ", "¨ ´ ˜", "﻿bom", "ǰ̣ ẞ ß", "test\u0085line sep",
]


def random_texts(n: int, seed: int, words=(3, 40)) -> list:
    rng = random.Random(seed)
    names = sorted(SCRIPTS)
    out = []
    for _ in range(n):
        ws = []
        for _ in range(rng.randint(*words)):
            r = rng.random()
            if r < 0.05:
                ws.append(rng.choice(EXTRAS))
                continue
            alpha = SCRIPTS[rng.choice(names)]
            w = "".join(rng.choice(alpha) for _ in range(rng.randint(1, 9)))
            if alpha in (SCRIPTS["cjk"], SCRIPTS["hiragana"]) and rng.random() < 0.5:
                w = "".join(rng.choice(alpha) for _ in range(rng.randint(10, 60)))     # CJK runs: long words
            ws.append(w)
        sep = rng.choice([" ", " ", " ", "  ", "\t", "\n", "　"])
        out.append(sep.join(ws) + rng.choice(["", ".", "!", " ?", "。"]))
    return out


@functools.lru_cache(maxsize=None)
def _trained(rule: str, vocab_size: int, seed: int):
    """(pieces [(piece, score)], charsmap bytes) of a Unigram model sentencepiece trains on the seeded corpus"""
    import sentencepiece as spm
    from sentencepiece import sentencepiece_model_pb2
    corpus = random_texts(6000 if vocab_size > 10000 else 3000, seed=seed) + UNIGRAM_TRAPS * 3
    f = io.BytesIO()
    spm.SentencePieceTrainer.train(sentence_iterator=iter(corpus), model_writer=f, vocab_size=vocab_size, model_type="unigram",
                                   hard_vocab_limit=False, normalization_rule_name=rule, character_coverage=0.9995,
                                   max_sentence_length=1 << 16, minloglevel=2, num_threads=4, seed_sentencepiece_size=200000)
    m = sentencepiece_model_pb2.ModelProto()
    m.ParseFromString(f.getvalue())
    return [(p.piece, p.score) for p in m.pieces], m.normalizer_spec.precompiled_charsmap


def charsmap_from_rules(rules: dict) -> bytes:
    """the precompiled_charsmap sentencepiece compiles from {source: target} normalization rules"""
    import sentencepiece as spm
    from sentencepiece import sentencepiece_model_pb2
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "rules.tsv")
        with open(path, "w") as f:
            for a, b in rules.items():
                f.write(" ".join(f"{ord(c):X}" for c in a) + "\t" + " ".join(f"{ord(c):X}" for c in b) + "\n")
        out = io.BytesIO()
        spm.SentencePieceTrainer.train(sentence_iterator=iter([f"a rule table line {i}" for i in range(200)]),
                                       model_writer=out, vocab_size=40, model_type="unigram", hard_vocab_limit=False,
                                       normalization_rule_tsv=path, minloglevel=2)
    m = sentencepiece_model_pb2.ModelProto()
    m.ParseFromString(out.getvalue())
    return m.normalizer_spec.precompiled_charsmap


def precompiled_charsmap(rule: str) -> bytes:
    return _trained(rule, 8000, 0)[1]


def _save(d: str, pieces, unk_id: int, charsmap, mask_lstrip: bool = True):
    """tokenizer.json of the XLM-RoBERTa shape (<s> <pad> </s> <unk> first, <mask> last) and its config, in d"""
    import base64
    vocab = [["<s>", 0.0], ["<pad>", 0.0], ["</s>", 0.0], ["<unk>", 0.0]]
    vocab += [[p, s] for p, s in pieces if p not in ("<s>", "<pad>", "</s>", "<unk>")] + [["<mask>", 0.0]]
    added = [dict(id=i, content=c, single_word=False, lstrip=(c == "<mask>" and mask_lstrip), rstrip=False, normalized=False,
                  special=True) for c, i in (("<s>", 0), ("<pad>", 1), ("</s>", 2), ("<unk>", 3), ("<mask>", len(vocab) - 1))]
    j = {
        "version": "1.0", "truncation": None, "padding": None, "added_tokens": added,
        "normalizer": {"type": "Precompiled", "precompiled_charsmap": base64.b64encode(charsmap).decode()} if charsmap else None,
        "pre_tokenizer": {"type": "Metaspace", "replacement": "▁", "prepend_scheme": "always", "split": True},
        "post_processor": {"type": "TemplateProcessing",
                           "single": [{"SpecialToken": {"id": "<s>", "type_id": 0}}, {"Sequence": {"id": "A", "type_id": 0}},
                                      {"SpecialToken": {"id": "</s>", "type_id": 0}}],
                           "pair": [{"SpecialToken": {"id": "<s>", "type_id": 0}}, {"Sequence": {"id": "A", "type_id": 0}},
                                    {"SpecialToken": {"id": "</s>", "type_id": 0}}, {"SpecialToken": {"id": "</s>", "type_id": 0}},
                                    {"Sequence": {"id": "B", "type_id": 0}}, {"SpecialToken": {"id": "</s>", "type_id": 0}}],
                           "special_tokens": {"<s>": {"id": "<s>", "ids": [0], "tokens": ["<s>"]},
                                              "</s>": {"id": "</s>", "ids": [2], "tokens": ["</s>"]}}},
        "decoder": {"type": "Metaspace", "replacement": "▁", "prepend_scheme": "always", "split": True},
        "model": {"type": "Unigram", "unk_id": unk_id if unk_id is not None else 3, "vocab": vocab, "byte_fallback": False},
    }
    with open(os.path.join(d, "tokenizer.json"), "w") as f:
        json.dump(j, f, ensure_ascii=False)
    with open(os.path.join(d, "tokenizer_config.json"), "w") as f:
        json.dump({"tokenizer_class": "XLMRobertaTokenizer", "model_max_length": 8192, "bos_token": "<s>", "eos_token": "</s>",
                   "cls_token": "<s>", "sep_token": "</s>", "pad_token": "<pad>", "unk_token": "<unk>",
                   "mask_token": "<mask>"}, f)
    return len(vocab)


def _load(pieces, charsmap, unk_id=3, mask_lstrip=True):
    from transformers import AutoTokenizer
    d = tempfile.mkdtemp(prefix="xlmr_tok_")
    _save(d, pieces, unk_id, charsmap, mask_lstrip)
    return AutoTokenizer.from_pretrained(d)


def make_unigram(rule: str = "nmt_nfkc", vocab_size: int = 8000, seed: int = 0):
    """an XLM-R-shaped tokenizer whose pieces and charsmap sentencepiece trained with `rule`, loaded by AutoTokenizer"""
    pieces, charsmap = _trained(rule, vocab_size, seed)
    return _load(pieces[3:], charsmap)                 # sentencepiece's own <unk> <s> </s> lead its pieces


def make_handmade(pieces, rule=None):
    """an XLM-R-shaped tokenizer with exactly these (piece, score) pairs after the four specials, and `rule`'s charsmap or no
    normalizer"""
    return _load(pieces, precompiled_charsmap(rule) if rule else None)


def save_pretrained_tokenizer(d: str, rule: str = "nmt_nfkc", vocab_size: int = 8000) -> int:
    """the tokenizer files of make_unigram in d (for a local checkpoint); returns the vocab size"""
    pieces, charsmap = _trained(rule, vocab_size, 0)
    return _save(d, pieces[3:], 3, charsmap)
