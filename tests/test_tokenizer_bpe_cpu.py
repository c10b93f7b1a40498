"""Device byte-level BPE tokenizer on the CPU: the codepoint classes against the installed `tokenizers` library, the split stage
and the whole kernels of csrc/tokenizer.cu through tests/cpu_shim against the library and the Hugging Face tokenizer call,
and which tokenizers are accepted."""
import itertools
import os
import subprocess
import tempfile

import numpy as np
import pytest

import bpe_corpus as bc
import tokenizer_corpus as tc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# White_Space in Unicode's PropList.txt, which Rust's char::is_whitespace follows
RUST_WHITESPACE = set(range(0x9, 0xE)) | {0x20, 0x85, 0xA0, 0x1680, 0x2028, 0x2029, 0x202F, 0x205F, 0x3000} | set(range(0x2000, 0x200B))


def test_bpe_classes_match_library_for_every_codepoint():
    """every codepoint but the surrogates, probed apart from how the tables were built: each codepoint between NUL separators
    in an isolated split (\\p{L}, \\p{N}, \\s), Rust whitespace against PropList's White_Space, and every contraction letter
    through the Llama-3 split itself ("'" + c is one piece exactly when c matches one of s t m d under (?i))"""
    from tokenizers import Regex, pre_tokenizers
    from adaptive_classifier_b200.tokenizer import (BPE_L, BPE_N, BPE_RUST, BPE_S, FOLD_LETTERS, LLAMA3_PATTERN, bpe_classes,
                                                    probe_codepoints)
    cls = bpe_classes()
    cps = [c for c in probe_codepoints().tolist() if c != 0]
    joined = "\0".join(map(chr, cps))
    for bit, pat in ((BPE_L, r"\p{L}"), (BPE_N, r"\p{N}"), (BPE_S, r"\s")):
        hit = {ord(p) for p, _ in pre_tokenizers.Split(Regex(pat), "isolated").pre_tokenize_str(joined) if len(p) == 1 and p != "\0"}
        bad = [hex(c) for c in cps if bool(cls[c] & bit) != (c in hit)]
        assert not bad, (pat, bad[:10])
    bad = [hex(c) for c in probe_codepoints().tolist() if bool(cls[c] & BPE_RUST) != (c in RUST_WHITESPACE)]
    assert not bad, bad[:10]
    split = pre_tokenizers.Split(Regex(LLAMA3_PATTERN), "isolated").pre_tokenize_str
    short = {FOLD_LETTERS.index(x) + 1 for x in "stmd"}
    # "'" + c + "z" starts with the piece "'" + c exactly when c is a contraction letter ("'cz" is one piece for any other
    # letter); a codepoint that is no letter matches none
    bad = [hex(c) for c in cps if (split("'" + chr(c) + "z")[0][0] == "'" + chr(c) if cls[c] & BPE_L else False)
           != ((cls[c] >> 4) in short)]
    assert not bad, bad[:10]
    assert not (cls[[c for c in cps if not cls[c] & BPE_L]] >> 4).any()
    for x, y in (("r", "e"), ("v", "e"), ("l", "l")):
        ix, iy = FOLD_LETTERS.index(x) + 1, FOLD_LETTERS.index(y) + 1
        firsts = [c for c in cps if cls[c] >> 4 == ix] + [ord("a")]
        seconds = [c for c in cps if cls[c] >> 4 == iy] + [ord("a")]
        for a in firsts:
            for b in seconds:
                w = "'" + chr(a) + chr(b)
                assert (split(w + "z")[0][0] == w) == (cls[a] >> 4 == ix and cls[b] >> 4 == iy), w
    assert cls[0x17F] >> 4 == FOLD_LETTERS.index("s") + 1                       # LATIN SMALL LETTER LONG S matches (?i)s


def _build(*extra):
    exe = os.path.join(tempfile.mkdtemp(prefix="bpe_emul_"), "tokenizer_bpe_emul")
    shim = os.path.join(ROOT, "tests", "cpu_shim")
    r = subprocess.run(["g++", "-std=c++17", "-O1", *extra, "-I/usr/local/cuda/include",
                        os.path.join(shim, "tokenizer_bpe_emul.cpp"), os.path.join(shim, "cuda_shim.cpp"), "-o", exe],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    return exe


@pytest.fixture(scope="module")
def emul():
    return _build()


def run_emul(exe, tok, texts, max_length, seed=1, mode=0):
    """mode 0: (tokens, lengths, max_len, ids, mask, type_ids); mode 1: (n_ent, entries [B, max_length - 2, 2])"""
    from adaptive_classifier_b200._cabi import bpe_spec_struct
    from adaptive_classifier_b200.tokenizer import bpe_spec
    spec, why = bpe_spec(tok)
    assert spec is not None, why
    _, (cls, vb, vo, vi, bi, mg, ab, ao, ai, af) = bpe_spec_struct(spec)
    n_added = len(spec["added"])
    if any(isinstance(t, bytes) for t in texts):
        enc = list(texts)
    else:
        enc = [t.encode("utf-8") for t in texts]
    to = np.cumsum([0] + [len(t) for t in enc]).astype(np.int64)
    d = tempfile.mkdtemp(prefix="bpe_run_")
    fin, fout = os.path.join(d, "in.bin"), os.path.join(d, "out.bin")
    with open(fin, "wb") as f:
        def rec(b):
            b = bytes(b)
            f.write(np.int64(len(b)).tobytes() + b + b"\0" * (-len(b) % 8))
        for a in (cls, vb[: vo[-1]], vo, vi, bi, mg[: len(spec["merges"])], ab[: ao[-1]], ao, ai[:n_added], af[:n_added]):
            rec(np.ascontiguousarray(a).tobytes())
        f.write(np.asarray([spec["split"], spec["prefix_space"], spec["ignore_merges"], spec["cls_id"], spec["sep_id"],
                            spec["pad_id"], len(texts), max_length, mode], dtype=np.int64).tobytes())
        rec(b"".join(enc))
        rec(to.tobytes())
    r = subprocess.run([exe, fin, fout, str(seed)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    out = np.fromfile(fout, dtype=np.int32)
    B, E = len(texts), max_length - 2
    if mode == 1:
        return out[:B], out[B:].reshape(B, E, 2)
    tokens = out[: B * max_length].reshape(B, max_length)
    lengths = out[B * max_length: B * max_length + B]
    max_len = out[B * max_length + B: B * max_length + B + 2]
    S = int(max_len[0])
    rest = out[B * max_length + B + 2:]
    ids, mask, tt = (rest[i * B * S:(i + 1) * B * S].reshape(B, S) for i in range(3))
    return tokens, lengths, max_len, ids, mask, tt


def device_rows(exe, tok, texts, max_length, seed=1):
    """the ids rows a BPETokenizer call produces: the kernels' rows, and the host tokenizer's for the texts they leave"""
    tokens, lengths, max_len, _, _, _ = run_emul(exe, tok, texts, max_length, seed)
    left = [i for i in range(len(texts)) if lengths[i] < 0]
    assert bool(left) == bool(max_len[1])
    host = tok([texts[i] for i in left], max_length=max_length, truncation=True)["input_ids"] if left else []
    rows = [tokens[i, : lengths[i]].tolist() for i in range(len(texts))]
    for i, r in zip(left, host):
        rows[i] = r
    return rows, left


def assert_same(exe, tok, texts, max_length, seed=1):
    """the kernels against tok(texts, max_length=..., truncation=True, padding=True), ids, mask and (absent) type ids"""
    ref = tok(texts, max_length=max_length, truncation=True, padding=True)
    tokens, lengths, max_len, ids, mask, tt = run_emul(exe, tok, texts, max_length, seed)
    want = ref["input_ids"]
    for i in range(len(texts)):
        if lengths[i] < 0:
            continue
        got = tokens[i, : lengths[i]].tolist()
        w = [x for x, m in zip(want[i], ref["attention_mask"][i]) if m]
        assert got == w, (repr(texts[i][:200]), got[:40], w[:40])
    kept = [i for i in range(len(texts)) if lengths[i] >= 0]
    if kept and max_len[1] == 0:
        assert ids.tolist() == want and mask.tolist() == ref["attention_mask"]
    assert "token_type_ids" not in ref
    return lengths


def _split_pieces(tok, texts, exe):
    """the split stage's words of each text as byte-level strings, as pre_tokenize_str shows them"""
    from adaptive_classifier_b200.tokenizer import byte_level_map
    inv = {b: s for s, b in byte_level_map().items()}
    n_ent, ent = run_emul(exe, tok, texts, 64, mode=1)
    out = []
    for t, n, e in zip(texts, n_ent, ent):
        raw = t.encode("utf-8")
        words = []
        for slot, info in e[:n]:
            assert info > 0
            nb, vp = info >> 1, info & 1
            start = slot - 1 + vp
            w = (b" " if vp else b"") + raw[start: start + nb - vp]
            words.append("".join(inv[x] for x in w))
        out.append(words)
    return out


ALPHABET = ["a", "É", "中", "1", "٣", "'", "s", "S", "L", "$", "-", " ", "\t", "\n", "\r", " ", "　"]


@pytest.mark.parametrize("kind", ["roberta", "roberta_prefix", "eurobert"])
def test_split_stage_matches_pre_tokenizer(emul, kind):
    """every string of up to 4 chars over representatives of each class (letters of three scripts, digits, the apostrophe and
    contraction letters in both cases, symbols, each kind of whitespace), and the trap corpus: the words of the split kernel
    equal pre_tokenize_str's pieces"""
    tok = bc.make_handmade(kind, [], added=False)
    pt = tok.backend_tokenizer.pre_tokenizer
    texts = ["".join(p) for n in range(1, 5) for p in itertools.product(ALPHABET, repeat=n)]
    texts += [t for t in bc.BPE_TRAPS if len(t) < 60 and "<" not in t and "[" not in t]
    got = _split_pieces(tok, texts, emul)
    bad = [(t, g, w) for t, g in zip(texts, got) if g != (w := [p for p, _ in pt.pre_tokenize_str(t)])]
    assert not bad, (len(bad), bad[:5])


@pytest.mark.parametrize("kind", bc.KINDS)
@pytest.mark.parametrize("vocab_size", [4000, 30000])
@pytest.mark.parametrize("max_length", [8, 128, 512, 8192])
def test_kernels_through_cpu_shim_match_hf(emul, kind, vocab_size, max_length):
    tok = bc.make_bpe(kind, vocab_size)
    texts = bc.BPE_TRAPS + tc.random_texts(30, seed=max_length) + [" ".join(tc.random_texts(30, seed=7))]
    if max_length == 8192:
        texts.append(" ".join(tc.random_texts(300, seed=5)))             # past 8192 tokens: truncated
    assert_same(emul, tok, texts, max_length)
    assert_same(emul, tok, texts[::-1], max_length, seed=12345)          # another thread order, another batch layout


@pytest.mark.parametrize("kind", ["roberta", "eurobert"])
def test_handmade_merge_lists(emul, kind):
    """ties (the leftmost pair first), runs of one symbol, a rank order in which a merge ranks before the merges that build
    its operands, and ignore_merges on words that are whole vocab entries no merge reaches"""
    runs = bc.make_handmade(kind, [("a", "a"), ("aa", "a"), ("b", "b"), ("bb", "bb")])
    texts = ["a" * n for n in range(1, 12)] + ["b" * n for n in range(1, 12)] + ["aaaa aaa", "abababa", "aab baa"]
    for t, w in (("aaaa", ["aa", "aa"]), ("aaa", ["aaa"])):
        assert runs.backend_tokenizer.encode(t, add_special_tokens=False).tokens == w
    assert_same(emul, runs, texts, 64)
    ties = bc.make_handmade(kind, [("x", "y"), ("y", "x"), ("y", "z"), ("z", "y")])
    assert_same(emul, ties, ["xyx", "yxy", "xyzyx", "zyxyz", "xyxyxyx", "yzyzy"], 32)
    nonmono = bc.make_handmade(kind, [("p", "qr"), ("pq", "r"), ("q", "r"), ("p", "q"), ("pqr", "pqr"), ("r", "p")])
    assert_same(emul, nonmono, ["pqr", "pqrpqr", "rpqr", "qrp", "pqpqr", "pqrrpqr"], 32)
    ig = bc.make_handmade(kind, [("e", "n"), ("en", "d")], extra=["endoftext", "Ġendoftext", "<s>", "endof"],
                          ignore_merges=True)
    assert ig.backend_tokenizer.encode("endoftext", add_special_tokens=False).ids == [ig.backend_tokenizer.token_to_id("endoftext")]
    assert_same(emul, ig, ["endoftext", "x endoftext endof end", "<s> endoftext<s>", "endoftexts"], 32)
    dup = bc.make_handmade(kind, [("c", "d"), ("d", "e"), ("c", "de"), ("cd", "e")], ignore_merges=False)
    assert_same(emul, dup, ["cde", "cdecde", "ccdee"], 32)


def test_added_token_semantics_pinned():
    """the library behaviours the kernel reproduces: normalized tokens only inside the gaps the others leave, lstrip taking
    whitespace, and the prefix space on every gap that does not start with one"""
    tok = bc.make_handmade("roberta", [("a", "b")], added=True)
    def enc(s):
        return tok.backend_tokenizer.encode(s, add_special_tokens=False)
    assert enc("zab<mask>").tokens == ["z", "ab", "<mask>"]
    assert enc("hi  \t<mask>").tokens == ["h", "i", "  \t<mask>"]
    pre = bc.make_handmade("roberta_prefix", [], added=True)
    assert pre.backend_tokenizer.encode("q<mask>r", add_special_tokens=False).tokens == ["Ġ", "q", "<mask>", "Ġ", "r"]


def test_huge_words_go_to_the_host(emul):
    """a text whose kept words include one longer than AC_BPE_MAX_WORD bytes (the space in front counted) is left to the
    host; words of exactly that many bytes, and long words past the kept ones, stay on the device; the composed rows equal
    the library's"""
    from adaptive_classifier_b200.tokenizer import MAX_WORD
    for kind in ("roberta_prefix", "eurobert"):
        tok = bc.make_bpe(kind)
        texts = ["x " + "a" * (MAX_WORD - 1), "x " + "a" * MAX_WORD, "a" * MAX_WORD, "a" * (MAX_WORD + 1), "a" * 1_000_000,
                 "ok " * 20 + "a" * 5000, "short text", "é" * 600]
        rows, left = device_rows(emul, tok, texts, 16)
        ref = tok(texts, max_length=16, truncation=True)["input_ids"]
        assert rows == ref
        assert left == ([1, 2, 3, 4, 7] if kind == "roberta_prefix" else [1, 3, 4, 7])   # " aaa…": one byte more


def test_kernels_under_address_sanitizer(monkeypatch):
    """a 1 MB word, 8192-token rows, words of AC_BPE_MAX_WORD and one more byte, and cut UTF-8, on a build with
    AddressSanitizer and a workspace of exactly the queried size"""
    from adaptive_classifier_b200.tokenizer import MAX_WORD
    exe = _build("-fsanitize=address", "-fno-omit-frame-pointer")
    monkeypatch.setenv("ASAN_OPTIONS", "detect_leaks=0")
    for kind in ("roberta_prefix", "eurobert", "modernbert"):
        tok = bc.make_bpe(kind)
        texts = ["a" * 1_000_000, " ".join(tc.random_texts(300, seed=5)), "a" * MAX_WORD, "a" * (MAX_WORD + 1),
                 " " + "é" * (MAX_WORD // 2), "x" * (MAX_WORD - 1)] + bc.BPE_TRAPS
        assert_same(exe, tok, texts, 8192)
        run_emul(exe, tok, [b"x \xe4\xb8", b"\xf0\x9f", b"\xe4", b"'"], 8)


@pytest.mark.parametrize("kind", bc.KINDS)
def test_bpe_tokenizers_are_accepted(kind):
    from adaptive_classifier_b200.tokenizer import SPLIT_GPT2, SPLIT_LLAMA3, bpe_spec, wordpiece_spec
    tok = bc.make_bpe(kind)
    spec, why = bpe_spec(tok)
    assert spec is not None, why
    assert spec["split"] == (SPLIT_LLAMA3 if kind == "eurobert" else SPLIT_GPT2)
    assert spec["prefix_space"] == (kind == "roberta_prefix") and spec["ignore_merges"] == (kind == "eurobert")
    assert not spec["type_ids"] and len(spec["byte_ids"]) == 256
    assert wordpiece_spec(tok)[0] is None


def _refused(tok, fragment):
    from adaptive_classifier_b200.tokenizer import bpe_spec
    spec, why = bpe_spec(tok)
    assert spec is None and fragment in why, why


def _with(kind, edit):
    import json
    from tokenizers import Tokenizer
    tok = bc.make_handmade(kind, [])
    j = json.loads(tok.backend_tokenizer.to_str())
    edit(j)
    return bc._wrap(Tokenizer.from_str(json.dumps(j)), kind)


def test_other_tokenizers_are_refused_with_a_reason():
    from tokenizers import AddedToken, Regex, normalizers, pre_tokenizers
    from transformers import RobertaTokenizer
    _refused(tc.make_tokenizer("bert"), "is not BPE")
    _refused(RobertaTokenizer(vocab={"<s>": 0, "<pad>": 1, "</s>": 2, "<unk>": 3, "a": 4}, merges=[]), "256 byte-level")
    _refused(_with("roberta", lambda j: j["model"].update(dropout=0.1)), "dropout")
    _refused(_with("roberta", lambda j: j["model"].update(continuing_subword_prefix="##")), "continuing_subword_prefix")
    _refused(_with("roberta", lambda j: j["model"].update(end_of_word_suffix="</w>")), "end_of_word_suffix")
    _refused(_with("roberta", lambda j: j["model"].update(byte_fallback=True)), "byte_fallback")
    _refused(_with("roberta", lambda j: j["pre_tokenizer"].update(use_regex=False)), "use_regex")
    _refused(_with("eurobert", lambda j: j["pre_tokenizer"]["pretokenizers"][0]["pattern"].update(
        Regex=bc.LLAMA3.replace("{1,3}", "+"))), "is not the Llama-3 pattern")
    _refused(_with("eurobert", lambda j: j["pre_tokenizer"]["pretokenizers"][0].update(behavior="Removed")), "Isolated")
    _refused(_with("eurobert", lambda j: j["pre_tokenizer"]["pretokenizers"][1].update(add_prefix_space=True)),
             "ByteLevel after Split")
    from tokenizers import processors
    t = bc.make_bpe("roberta")
    t.backend_tokenizer.post_processor = processors.ByteLevel()
    _refused(t, "post_processor 'ByteLevel'")
    t = bc.make_bpe("roberta")
    t.backend_tokenizer.post_processor = processors.TemplateProcessing(single="<s> $A", special_tokens=[("<s>", 0)])
    _refused(t, "template")
    t = bc.make_bpe("roberta")
    t.backend_tokenizer.normalizer = normalizers.NFC()
    _refused(t, "normalizer")
    t = bc.make_bpe("roberta")
    t.backend_tokenizer.pre_tokenizer = pre_tokenizers.Whitespace()
    _refused(t, "pre_tokenizer")
    t = bc.make_bpe("roberta")
    t.backend_tokenizer.pre_tokenizer = pre_tokenizers.Sequence([pre_tokenizers.Split(Regex(r"\s+"), "isolated"),
                                                                 pre_tokenizers.ByteLevel(use_regex=False)])
    _refused(t, "is not the Llama-3 pattern")
    t = bc.make_bpe("roberta")
    t.add_tokens([AddedToken("foo", single_word=True)])
    _refused(t, "single_word=True")
    t = bc.make_bpe("modernbert")
    t.add_tokens([AddedToken("<r>", normalized=True, rstrip=True)])
    _refused(t, "rstrip")
    t = bc.make_bpe("roberta")
    t.truncation_side = "left"
    _refused(t, "left")
    t = bc.make_bpe("roberta")
    t.padding_side = "left"
    _refused(t, "left")
    t = bc.make_bpe("roberta")
    t.backend_tokenizer.encode_special_tokens = True
    _refused(t, "encode_special_tokens")
