"""Device WordPiece tokenizer on the CPU: the Unicode tables against the installed `tokenizers` library codepoint by codepoint,
the kernels of csrc/tokenizer.cu through tests/cpu_shim against the Hugging Face tokenizer call, and which tokenizers are
accepted."""
import itertools
import os
import subprocess
import tempfile

import numpy as np
import pytest

import tokenizer_corpus as tc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FLAGS = list(itertools.product([False, True], repeat=4))     # clean_text, handle_chinese_chars, strip_accents, lowercase


@pytest.mark.parametrize("flags", FLAGS, ids=lambda f: "".join(k if v else "-" for k, v in zip("CZSL", f)))
def test_tables_match_library_for_every_codepoint(flags):
    """every codepoint but the surrogates: the table's expansion equals normalize_str of the codepoint alone (one library
    call per codepoint, not the batched probe the tables are built from)"""
    from tokenizers import normalizers
    from adaptive_classifier_b200.tokenizer import IDENTITY, probe_codepoints, unicode_tables
    norm, _, pool = unicode_tables(*flags)
    nz = normalizers.BertNormalizer(clean_text=flags[0], handle_chinese_chars=flags[1], strip_accents=flags[2],
                                    lowercase=flags[3])
    f = nz.normalize_str
    bad = []
    for c in probe_codepoints().tolist():
        e = int(norm[c])
        got = chr(c) if e & IDENTITY else "".join(map(chr, pool[(e & 0x3FFFFFFF) >> 5:((e & 0x3FFFFFFF) >> 5) + (e & 31)]))
        if got != f(chr(c)):
            bad.append(c)
    assert not bad, f"{len(bad)} codepoints differ, first {[hex(c) for c in bad[:10]]}"


def test_pretokenizer_classes_every_codepoint():
    """every codepoint but the surrogates: its class equals what BertPreTokenizer makes of 'a' + c + 'a' (one piece: part of a
    word, two: dropped whitespace, three: punctuation)"""
    from tokenizers import pre_tokenizers
    from adaptive_classifier_b200.tokenizer import OTHER, PUNCT, SPACE, probe_codepoints, pretokenizer_classes
    cls = pretokenizer_classes()
    pt = pre_tokenizers.BertPreTokenizer().pre_tokenize_str
    want = {1: OTHER, 2: SPACE, 3: PUNCT}
    bad = [c for c in probe_codepoints().tolist() if want[len(pt("a" + chr(c) + "a"))] != cls[c]]
    assert not bad, [hex(c) for c in bad[:10]]
    assert all(cls[ord(c)] == PUNCT for c in "$+<=>^`|~")        # ASCII punctuation to the library, symbols to Unicode


def test_canonical_reordering_recorded():
    """the library reorders U+1D16D U+1D165 (classes 226, 216) when strip_accents runs NFD, across a removed ZWSP and a stripped
    U+0301, not across U+034F (combining grapheme joiner, class 0): the tables carry ranks and a blocker for exactly that"""
    from tokenizers import normalizers
    from adaptive_classifier_b200.tokenizer import BLOCKER, unicode_tables
    nz = normalizers.BertNormalizer(lowercase=True)
    a, b = "\U0001D16D", "\U0001D165"
    assert nz.normalize_str(a + b) == b + a and nz.normalize_str(a + "​" + b) == b + a
    assert nz.normalize_str(a + "͏" + b) == a + b and nz.normalize_str(a + "́" + b) == b + a
    norm, cls, _ = unicode_tables(True, True, True, True)
    assert (cls[0x1D16D] >> 2) > (cls[0x1D165] >> 2) > 0 and norm[0x34F] & BLOCKER and not norm[0x301] & BLOCKER
    assert not norm[0x200B] & BLOCKER
    _, cls_cased, _ = unicode_tables(True, True, False, False)
    assert (cls_cased >> 2).max() == 0                             # no NFD, no reordering


def test_reorder_model_matches_library_for_every_pair():
    """for every ordered pair (a, b) of the codepoints unicodedata calls combining and that survive normalization, the
    kernel's rule (b moves before a when 0 < rank(b) < rank(a)) gives what normalize_str(a + b) gives; and for every removed
    codepoint NFD sees, the blocker bit says whether U+1D16D c U+1D165 keeps its order"""
    import unicodedata
    from tokenizers import normalizers
    from adaptive_classifier_b200.tokenizer import BLOCKER, IDENTITY, probe_codepoints, unicode_tables
    for flags in ((True, True, True, True), (False, False, True, False)):
        norm, cls, _ = unicode_tables(*flags)
        nz = normalizers.BertNormalizer(clean_text=flags[0], handle_chinese_chars=flags[1], strip_accents=True,
                                        lowercase=flags[3])
        cps = probe_codepoints()
        ident = cps[(norm[cps] & IDENTITY) != 0]
        marks = [int(c) for c in ident if unicodedata.combining(chr(c)) or cls[c] >> 2]
        assert len(marks) > 100
        rank = {c: int(cls[c]) >> 2 for c in marks}
        bad = []
        for a in marks:
            for b in marks:
                want = chr(b) + chr(a) if 0 < rank[b] < rank[a] else chr(a) + chr(b)
                if nz.normalize_str(chr(a) + chr(b)) != want:
                    bad.append((hex(a), hex(b)))
        assert not bad, bad[:10]
        A, B = "\U0001D16D", "\U0001D165"
        empty = [int(c) for c in cps if not norm[c] & IDENTITY and not norm[c] & 31]
        bad = [hex(c) for c in empty if (nz.normalize_str(A + chr(c) + B) == A + B) != bool(norm[c] & BLOCKER)]
        assert not bad, bad[:10]


def _build_emul(*extra):
    exe = os.path.join(tempfile.mkdtemp(prefix="tok_emul_"), "tokenizer_emul")
    shim = os.path.join(ROOT, "tests", "cpu_shim")
    r = subprocess.run(["g++", "-std=c++17", "-O1", *extra, "-I/usr/local/cuda/include", os.path.join(shim, "tokenizer_emul.cpp"),
                        os.path.join(shim, "cuda_shim.cpp"), "-o", exe], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    return exe


@pytest.fixture(scope="module")
def emul():
    return _build_emul()


def run_emul(exe, tok, texts, max_length, seed=1):
    from adaptive_classifier_b200._cabi import tokenizer_spec_struct
    from adaptive_classifier_b200.tokenizer import pack_strings, wordpiece_spec
    spec, why = wordpiece_spec(tok)
    assert spec is not None, why
    _, (norm, cls, pool, vb, vo, vi, ab, ao, ai) = tokenizer_spec_struct(spec)
    if not spec["added"]:
        ab, ao, ai = np.zeros(0, np.uint8), np.zeros(1, np.int64), np.zeros(0, np.int32)
    if any(isinstance(t, bytes) for t in texts):
        to = np.cumsum([0] + [len(t) for t in texts]).astype(np.int64)
        tb = np.frombuffer(b"".join(texts) + b"\0", dtype=np.uint8)
    else:
        tb, to = pack_strings(texts)
    d = tempfile.mkdtemp(prefix="tok_run_")
    fin, fout = os.path.join(d, "in.bin"), os.path.join(d, "out.bin")
    with open(fin, "wb") as f:
        def rec(b):
            b = bytes(b)
            f.write(np.int64(len(b)).tobytes() + b + b"\0" * (-len(b) % 8))
        for a in (norm, cls, pool, vb[: vo[-1]], vo, vi, ab[: ao[-1]], ao, ai[: len(spec["added"])]):
            rec(np.ascontiguousarray(a).tobytes())
        rec(spec["prefix"])
        f.write(np.asarray([spec["cls_id"], spec["sep_id"], spec["pad_id"], spec["unk_id"], spec["max_input_chars"],
                            len(texts), max_length], dtype=np.int64).tobytes())
        rec(tb[: to[-1]].tobytes())
        rec(to.tobytes())
    r = subprocess.run([exe, fin, fout, str(seed)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    out = np.fromfile(fout, dtype=np.int32)
    B = len(texts)
    S = int(out[B * max_length + B])
    rest = out[B * max_length + B + 1:]
    ids, mask, tt = (rest[i * B * S:(i + 1) * B * S].reshape(B, S) for i in range(3))
    return ids, mask, (tt if spec["type_ids"] else None)


def assert_same(exe, tok, texts, max_length, seed=1):
    ids, mask, tt = run_emul(exe, tok, texts, max_length, seed)
    ref = tok(texts, max_length=max_length, truncation=True, padding=True)
    want = np.asarray(ref["input_ids"], dtype=np.int32)
    for i in range(len(texts)):
        assert ids[i].tolist() == want[i].tolist(), (repr(texts[i][:200]), ids[i].tolist()[:40], want[i].tolist()[:40])
    assert np.array_equal(mask, np.asarray(ref["attention_mask"], dtype=np.int32))
    if "token_type_ids" in ref:
        assert tt is not None and np.array_equal(tt, np.asarray(ref["token_type_ids"], dtype=np.int32))
    else:
        assert tt is None


@pytest.mark.parametrize("kind", ["bert", "bert_cased", "electra", "mpnet"])
@pytest.mark.parametrize("max_length", [8, 128, 512])
def test_kernel_through_cpu_shim_matches_hf(emul, kind, max_length):
    tok = tc.make_tokenizer(kind)
    texts = tc.TRAPS + tc.random_texts(40, seed=max_length) + [" ".join(tc.random_texts(30, seed=7))]
    assert_same(emul, tok, texts, max_length)
    assert_same(emul, tok, texts[::-1], max_length, seed=12345)    # another thread order, another batch layout


def test_kernel_short_batches_and_huge_word(emul):
    tok = tc.make_tokenizer("bert")
    assert_same(emul, tok, ["hi"], 128)
    assert_same(emul, tok, ["", "a"], 8)
    assert_same(emul, tok, ["a" * 1_000_000, "x " + "é" * 300_000 + " y"], 16)


def test_invalid_utf8_stays_inside_the_text(emul):
    """bytes Python never produces (a cut sequence at the end of the last text, a lead byte past 0xF4, a stray continuation
    byte, an encoded value past U+10FFFF) are read as U+FFFD, which clean_text removes"""
    tok = tc.make_tokenizer("bert")
    texts = [b"hello \xf5 world \x80", b"hello \xf4\x90\x80\x80 world", b"hello world \xe4\xb8"]
    ids, mask, _ = run_emul(emul, tok, texts, 16)
    want = tok(["hello  world"] * 3, max_length=16, truncation=True, padding=True)
    assert ids.tolist() == want["input_ids"] and mask.tolist() == want["attention_mask"]


def test_kernel_under_address_sanitizer(monkeypatch):
    """the per-thread workspace indexing (a 1 MB word, 8192-token rows, words at max_input_chars_per_word) and the bounded
    UTF-8 decode on a build with AddressSanitizer: every host buffer is exactly as large as the kernel may touch"""
    exe = _build_emul("-fsanitize=address", "-fno-omit-frame-pointer")
    monkeypatch.setenv("ASAN_OPTIONS", "detect_leaks=0")       # the shim keeps its shared-memory pool for the process
    tok = tc.make_tokenizer("bert")
    texts = ["a" * 1_000_000, " ".join(tc.random_texts(400, seed=5)), "é" * 100, "é" * 101] + tc.TRAPS
    assert_same(exe, tok, texts, 8192)
    run_emul(exe, tok, [b"x \xe4\xb8", b"\xf0\x9f"], 8)


def test_tokenizer_json_truncation_and_padding_fields_are_overridden(emul):
    tok = tc.make_tokenizer("bert")
    tok.backend_tokenizer.enable_truncation(max_length=5)
    tok.backend_tokenizer.enable_padding(length=40, pad_id=tok.pad_token_id, pad_token=tok.pad_token)
    assert_same(emul, tok, tc.TRAPS[:8], 64)


@pytest.mark.parametrize("kind", ["bert", "bert_cased", "electra", "mpnet"])
def test_wordpiece_tokenizers_are_accepted(kind):
    from adaptive_classifier_b200.tokenizer import wordpiece_spec
    spec, why = wordpiece_spec(tc.make_tokenizer(kind))
    assert spec is not None, why
    assert spec["type_ids"] == (kind != "mpnet")
    assert spec["flags"][3] == (kind != "bert_cased")


def _refused(tok, fragment):
    from adaptive_classifier_b200.tokenizer import wordpiece_spec
    spec, why = wordpiece_spec(tok)
    assert spec is None and fragment in why, why


def test_other_tokenizers_are_refused_with_a_reason():
    from tokenizers import normalizers
    from transformers import AlbertTokenizer, RobertaTokenizer, XLMRobertaTokenizer
    _refused(RobertaTokenizer(vocab={"<s>": 0, "<pad>": 1, "</s>": 2, "<unk>": 3, "a": 4}, merges=[]), "BPE")
    uni = [("<s>", 0.0), ("<pad>", 0.0), ("</s>", 0.0), ("<unk>", 0.0), ("▁a", -1.0)]
    _refused(XLMRobertaTokenizer(vocab=uni), "Unigram")
    _refused(AlbertTokenizer(vocab=[("<pad>", 0.0), ("<unk>", 0.0), ("[CLS]", 0.0), ("[SEP]", 0.0), ("▁a", -1.0)]), "Unigram")
    from test_deberta_cpu import deberta_tokenizer_words
    _refused(deberta_tokenizer_words(["a", "b"]), "Unigram")
    t = tc.make_tokenizer("bert")
    t.backend_tokenizer.normalizer = normalizers.Sequence([normalizers.NFD(), normalizers.Lowercase()])
    _refused(t, "Sequence")
    t = tc.make_tokenizer("bert")
    from tokenizers import AddedToken
    t.add_tokens([AddedToken("foo", single_word=True, normalized=False)])
    _refused(t, "single_word=True")
    from transformers import BertTokenizerFast
    _refused(BertTokenizerFast(vocab={w: i for i, w in enumerate(tc.SPECIALS_BERT + ["", "a"])}), "empty entry")
    t = tc.make_tokenizer("bert")
    t.truncation_side = "left"
    _refused(t, "left")
    t = tc.make_tokenizer("bert")
    t.padding_side = "left"
    _refused(t, "left")
