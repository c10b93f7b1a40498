"""Seeded WordPiece tokenizers and the trap corpus shared by the CPU (cpu_shim) and GPU tests of the device tokenizer."""
import random

SPECIALS_BERT = ["[PAD]", "[UNK]", "[CLS]", "[SEP]", "[MASK]"]
SPECIALS_MPNET = ["<s>", "<pad>", "</s>", "[UNK]", "<mask>"]
LETTERS = "abcdefghijklmnopqrstuvwxyzABCDEFGHIJKLMNOPQRSTUVWXYZéèüößçñøåæœıσςπλ中文字한국어д"


MARKS = ["\U0001D165", "\U0001D16D", "\u1AC1", "\u0C3C", "\u0898"]


def seeded_vocab(specials, seed: int = 0, n_words: int = 600) -> list:
    """specials, every single char of LETTERS and digits / ASCII punctuation with and without '##', seeded words and their
    '##' tails (multi-byte pieces included), a few whole words of the corpus"""
    rng = random.Random(seed)
    singles = list(LETTERS) + list("0123456789") + list("!\"#$%&'()*+,-./:;<=>?@[\\]^_`{|}~")
    vocab = list(specials) + singles + ["##" + c for c in singles]
    for _ in range(n_words):
        w = "".join(rng.choice(LETTERS[:60]) for _ in range(rng.randint(2, 7)))
        vocab += [w, "##" + w[1:], "##" + w[-2:]]
    vocab += ["hello", "world", "##s", "un", "##aff", "##able", "cafe", "café", "##é", "naive", "istanbul", "σοφος",
              "ὀδυσσευς", "mask", "cls"]
    # marks the library orders (U+1D165 class 216, U+1D16D class 226) next to marks newer than its Unicode tables, which it
    # treats as starters (U+1AC1, U+0C3C, U+0898)
    vocab += ["x", "##" + MARKS[0], "##" + MARKS[1]] + ["##" + m for m in MARKS[2:]] + [m for m in MARKS]
    seen, out = set(), []
    for w in vocab:
        if w not in seen:
            seen.add(w)
            out.append(w)
    return out


def make_tokenizer(kind: str, seed: int = 0):
    """'bert' (uncased), 'bert_cased', 'electra' or 'mpnet', built in memory from a seeded vocab"""
    from transformers import BertTokenizerFast, ElectraTokenizer, MPNetTokenizer
    if kind == "mpnet":
        return MPNetTokenizer(vocab={w: i for i, w in enumerate(seeded_vocab(SPECIALS_MPNET, seed))})
    vocab = {w: i for i, w in enumerate(seeded_vocab(SPECIALS_BERT, seed))}
    if kind == "electra":
        return ElectraTokenizer(vocab=vocab, do_lower_case=True)
    return BertTokenizerFast(vocab=vocab, do_lower_case=(kind == "bert"))


TRAPS = [
    "hello [MASK] world", "[mask] and [cls] stay text", "[MASK][SEP][CLS]x[PAD]", "hello <mask> world", "x   <mask>y",
    "a" * 100, "a" * 101, "é" * 100, "é" * 101, "b" * 99 + "中", "helloworld☃", "un☃able", "unaffable", "",
    "\x00a�b​c\td\ne\rf\x07g h", "\x00�​\x7f",
    "ΣΟΦΟΣ ὈΔΥΣΣΕΎΣ σς", "İstanbul İ", "한국어 한", "ȩ́ ä́ Ǖ",
    "x\U0001D16D\U0001D165 x\U0001D165\U0001D16D x\U0001D16D͏\U0001D165 x\U0001D16D​\U0001D165 x\U0001D16D́\U0001D165",
    "\U0001D15F\U0001D160 \U0001D1BB", "中文字符 𠀀𪜀 \U00030000\U00031350 㐀 豈",
    "emoji 👩‍👩‍👧 a b c　d", "$ + < = > ^ ` | ~ a$b+c<d=e>f^g`h|i~j", "¡¿«»—…·",
    "Café NAÏVE naïve Ⅻ ﬁ ＡＢＣ",
    "x\U0001D16D\u1AC1 x\u1AC1\U0001D16D x\U0001D16D\u1AC1\U0001D165 x\U0001D16D\u0C3C\U0001D165 x\u0898\U0001D16D\U0001D165",
    "\U0001D16D\U0001D165\u1AC1\U0001D16D\U0001D165 x\U0001D16D\u0301\u1AC1\U0001D165",
]


def random_texts(n: int, seed: int, words=(2, 40)) -> list:
    """seeded mixed-script texts: ASCII / accented / Greek / Cyrillic / CJK / Hangul words, punctuation, specials, spaces"""
    rng = random.Random(seed)
    pool = LETTERS + "ÀÉÎÕÜàéîõüĀāŠšЖжΩωابت" + "́̈" + "😀🎉"
    out = []
    for _ in range(n):
        ws = []
        for _ in range(rng.randint(*words)):
            r = rng.random()
            if r < 0.05:
                ws.append(rng.choice(["[MASK]", "<mask>", "[SEP]", ",", ".", "!", "中国", "\t", "　"]))
            else:
                ws.append("".join(rng.choice(pool) for _ in range(rng.randint(1, 9))))
        out.append(rng.choice([" ", "  ", " \n"]).join(ws))
    return out
