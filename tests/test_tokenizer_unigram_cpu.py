"""Device SentencePiece Unigram tokenizer on the CPU: the charsmap decoder and grapheme classes against the installed
`tokenizers` library, the Precompiled stage and the whole kernels of csrc/tokenizer.cu through tests/cpu_shim against the
library and the Hugging Face tokenizer call, and which tokenizers are accepted."""
import json
import os
import subprocess
import tempfile

import numpy as np
import pytest

import unigram_corpus as uc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _build(*extra):
    exe = os.path.join(tempfile.mkdtemp(prefix="unigram_emul_"), "tokenizer_unigram_emul")
    shim = os.path.join(ROOT, "tests", "cpu_shim")
    r = subprocess.run(["g++", "-std=c++17", "-O1", *extra, "-I/usr/local/cuda/include",
                        os.path.join(shim, "tokenizer_unigram_emul.cpp"), os.path.join(shim, "cuda_shim.cpp"), "-o", exe],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    return exe


@pytest.fixture(scope="module")
def emul():
    return _build()


def _spec(tok):
    from adaptive_classifier_b200.tokenizer import unigram_spec
    spec, why = unigram_spec(tok)
    assert spec is not None, why
    return spec


def run_emul(exe, spec, texts, max_length, seed=1, mode=0):
    """mode 0: (tokens, lengths, max_len, ids, mask); mode 1: the Precompiled output of each text (None: over the workspace)"""
    from adaptive_classifier_b200._cabi import unigram_spec_struct
    _, (cls, mk, mko, mv, mvo, pb, po, ps, ab, ao, ai, af) = unigram_spec_struct(spec)
    n_added = len(spec["added"])
    enc = [t if isinstance(t, bytes) else t.encode("utf-8") for t in texts]
    to = np.cumsum([0] + [len(t) for t in enc]).astype(np.int64)
    d = tempfile.mkdtemp(prefix="unigram_run_")
    fin, fout = os.path.join(d, "in.bin"), os.path.join(d, "out.bin")
    with open(fin, "wb") as f:
        def rec(b):
            b = bytes(b)
            f.write(np.int64(len(b)).tobytes() + b + b"\0" * (-len(b) % 8))
        for a in (cls, mk[: mko[-1]], mko, mv[: mvo[-1]], mvo, pb[: po[-1]], po, ps, ab[: ao[-1]], ao, ai[:n_added],
                  af[:n_added]):
            rec(np.ascontiguousarray(a).tobytes())
        f.write(np.asarray([spec["grow"], spec["unk_id"], spec["cls_id"], spec["sep_id"], spec["pad_id"], len(texts),
                            max_length, mode], dtype=np.int64).tobytes())
        rec(b"".join(enc))
        rec(to.tobytes())
    r = subprocess.run([exe, fin, fout, str(seed)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    raw = open(fout, "rb").read()
    if mode == 1:
        out, at = [], 0
        for _ in texts:
            n = int(np.frombuffer(raw, dtype=np.int64, count=1, offset=at)[0])
            at += 8
            out.append(None if n < 0 else raw[at:at + n].decode("utf-8"))
            at += max(n, 0)
        return out
    out = np.frombuffer(raw, dtype=np.int32)
    B = len(texts)
    tokens = out[: B * max_length].reshape(B, max_length)
    lengths = out[B * max_length: B * max_length + B]
    max_len = out[B * max_length + B: B * max_length + B + 2]
    S = int(max_len[0])
    rest = out[B * max_length + B + 2:]
    ids, mask = (rest[i * B * S:(i + 1) * B * S].reshape(B, S) for i in range(2))
    return tokens, lengths, max_len, ids, mask


def assert_same(exe, tok, texts, max_length, seed=1):
    """the kernels against tok(texts, max_length=..., truncation=True, padding=True); returns the texts left to the host"""
    ref = tok(texts, max_length=max_length, truncation=True, padding=True)
    tokens, lengths, max_len, ids, mask = run_emul(exe, _spec(tok), texts, max_length, seed)
    want = ref["input_ids"]
    left = [i for i in range(len(texts)) if lengths[i] < 0]
    assert bool(left) == bool(max_len[1])
    for i in range(len(texts)):
        if lengths[i] < 0:
            continue
        got = tokens[i, : lengths[i]].tolist()
        w = [x for x, m in zip(want[i], ref["attention_mask"][i]) if m]
        assert got == w, (repr(texts[i][:200]), got[:40], w[:40])
    if not left:
        assert ids.tolist() == want and mask.tolist() == ref["attention_mask"]
    assert "token_type_ids" not in ref
    return left


def _precompiled_reference(pairs, s: str) -> str:
    """Precompiled as the library documents it, on extended grapheme clusters cut by the `regex` module's \\X (independent of
    the class table the kernels read): a cluster shorter than 6 bytes that a key is a prefix of becomes the shortest such
    key's value; otherwise each char its own value, or itself"""
    import regex
    out = []
    for g in regex.findall(r"\X", s):
        b = g.encode()
        hit = next((pairs[b[:n]] for n in range(1, len(b) + 1) if b[:n] in pairs), None) if len(b) < 6 else None
        out.append(hit.decode() if hit is not None else "".join(pairs.get(c.encode(), c.encode()).decode() for c in g))
    return "".join(out)


@pytest.mark.parametrize("rule", uc.RULES)
def test_decoded_charsmap_matches_normalize_str(rule):
    """every decoded pair against the library: normalize_str(key) is what Precompiled makes of the key from the decoded
    pairs, on clusters cut by another implementation of the Unicode rules, not read from the class table the kernels use"""
    from tokenizers import normalizers
    from adaptive_classifier_b200.tokenizer import charsmap_tables
    blob = uc.precompiled_charsmap(rule)
    tables = charsmap_tables(blob)
    pairs = dict(tables["pairs"])
    assert len(pairs) > 200000 and tables["grow"] == max(-(-len(v) // len(k)) for k, v in pairs.items())
    nz = normalizers.Precompiled(blob)
    bad = []
    for k in pairs:
        s = k.decode("utf-8")
        want = _precompiled_reference(pairs, s)
        if nz.normalize_str(s) != want:
            bad.append((s, nz.normalize_str(s), want))
    assert not bad, (len(bad), bad[:5])


def test_grapheme_classes_pinned():
    """the probe's counts, and the classes of a few codepoints each rule needs"""
    from adaptive_classifier_b200.tokenizer import BPE_RUST, G_CONTROL, G_JOIN, G_PREPEND, unigram_classes
    cls = unigram_classes()
    assert int(((cls & G_JOIN) > 0).sum()) == 2577
    assert cls[0x301] & G_JOIN and cls[0x200D] & G_JOIN and cls[0x93F] & G_JOIN          # Extend, ZWJ, SpacingMark
    assert cls[0xD] & G_CONTROL and cls[0xA] & G_CONTROL and cls[0x200B] & G_CONTROL and not cls[ord("a")] & G_CONTROL
    assert cls[0x600] & G_PREPEND and not cls[ord("a")] & G_PREPEND
    assert cls[0x3000] & BPE_RUST and cls[0x85] & BPE_RUST and not cls[0x200B] & BPE_RUST
    # printable ASCII, the probe charsmap's own target letter 'b' among it, is no control, joins nothing and is no Prepend
    assert not any(cls[c] & (G_JOIN | G_CONTROL | G_PREPEND) for c in range(0x20, 0x7F)), \
        [chr(c) for c in range(0x20, 0x7F) if cls[c] & 7]
    assert all(cls[c] & G_CONTROL for c in list(range(0, 0x20)) + [0x7F])


def test_grapheme_classes_against_the_library():
    """the classes decide cluster cuts as the library does on each probe string, the mapping target and NUL included"""
    from tokenizers import normalizers
    from adaptive_classifier_b200.tokenizer import G_CONTROL, G_JOIN, G_PREPEND, all_to_b_charsmap, unigram_classes
    cls = unigram_classes()
    probe = normalizers.Precompiled(all_to_b_charsmap())
    for base in ("a", "b", "x", "\0", "\t", "ǅ", "ｆ"):
        for mark in ("\u0301", "\u0307", "\u0323", "\u200d", "\u093f"):
            if len((base + mark).encode()) >= 6:
                continue                          # normalized char by char whatever its clusters: the probe cannot see them
            joined = len(probe.normalize_str(base + mark)) == 1
            assert joined == (bool(cls[ord(mark)] & G_JOIN) and not cls[ord(base)] & G_CONTROL), ascii(base + mark)
    assert len(probe.normalize_str("\u0600b")) == 1 and cls[0x600] & G_PREPEND


def _norm_probe_texts(rule: str):
    """every codepoint alone, after mapped bases of 1, 2 and 3 bytes, and before 'x'; CR LF; clusters of 5 and 6 bytes.  The
    1-byte bases: 'b', which starts keys of every rule (b + U+0307 -> U+1E03 ...), and TAB, a key of its own under nmt_nfkc
    and nmt_nfkc_cf (nfkc maps no 1-byte char)"""
    from adaptive_classifier_b200.tokenizer import charsmap_tables, probe_codepoints
    pairs = dict(charsmap_tables(uc.precompiled_charsmap(rule))["pairs"])
    assert any(k.startswith(b"b") and len(k) > 1 for k in pairs)
    assert (b"\t" in pairs) == (rule != "nfkc") and "ǅ".encode() in pairs and "ｆ".encode() in pairs
    chars = [chr(c) for c in probe_codepoints().tolist()]
    texts = list(chars)
    for base in ["b", "ǅ", "ｆ"] + (["\t"] if rule != "nfkc" else []):
        texts += [base + c for c in chars]
    texts += [c + "x" for c in chars]
    texts += ["\r\n", "\r\r\n\n", "x\r\ny", "Ａ́", "①́", "ｆ́x", "ｆ̈́", "ｆ‍", "ｆि", "a" + "́" * 2, "ǅ́́",
              "b\u0307", "b\u0323", "ab\u0307c", "abb\u0323a b\u0307", "B\u0307\u0323"]
    return texts


@pytest.mark.parametrize("rule", uc.RULES)
def test_precompiled_stage_matches_normalize_str(emul, rule):
    from tokenizers import normalizers
    tok = uc.make_unigram(rule)
    spec = _spec(tok)
    nz = normalizers.Precompiled(uc.precompiled_charsmap(rule))
    texts = _norm_probe_texts(rule)
    got = []
    for i in range(0, len(texts), 200000):
        got += run_emul(emul, spec, texts[i:i + 200000], 8, mode=1)
    bad = [(t, g, w) for t, g in zip(texts, got) if g != (w := nz.normalize_str(t))]
    assert not bad, (len(bad), [tuple(map(ascii, b)) for b in bad[:5]])


@pytest.mark.parametrize("rule", uc.RULES)
@pytest.mark.parametrize("vocab_size", [8000, 30000])
@pytest.mark.parametrize("max_length", [8, 128, 512, 8192])
def test_kernels_through_cpu_shim_match_hf(emul, rule, vocab_size, max_length):
    tok = uc.make_unigram(rule, vocab_size)
    texts = uc.UNIGRAM_TRAPS + uc.random_texts(30, seed=max_length) + [" ".join(uc.random_texts(30, seed=7))]
    if max_length == 8192:
        texts.append(" ".join(uc.random_texts(300, seed=5)))            # past 8192 tokens: truncated
    left = assert_same(emul, tok, texts, max_length)
    assert assert_same(emul, tok, texts[::-1], max_length, seed=12345) == [len(texts) - 1 - i for i in left][::-1]
    assert len(left) <= 2


def test_handmade_lattices(emul):
    """score ties (the first candidate kept), fused unknown chars, the special pieces as plain text, '▁' in the text, and
    added tokens with lstrip"""
    ties = uc.make_handmade([("▁", -1.0), ("a", -2.0), ("b", -2.0), ("ab", -4.0), ("▁ab", -5.0), ("▁a", -3.0), ("x", -9.0),
                             ("y", -9.0), ("xy", -18.0), ("▁x", -9.0)])
    enc = ties.backend_tokenizer.encode
    texts = ["ab", "abab", "aab", "xy", "xyxy", "zzz", "qzq", "a qqq b", "ééé a", "▁ab", "a▁▁b", "<s>ab</s>", "x <mask>",
             "ab  <mask>", "<mask>ab", "<unk>", "▁<unk>", "q<s>q", "<pad>"]
    assert assert_same(emul, ties, texts, 32) == []
    for t, w in (("zzz", ["▁", "zzz"]), ("qzq", ["▁", "qzq"])):
        assert enc(t, add_special_tokens=False).tokens == w, enc(t, add_special_tokens=False).tokens
    norm = uc.make_handmade([("▁", -1.0), ("A", -1.0), ("1", -1.0), ("fx", -1.0), ("▁fx", -0.5)], rule="nmt_nfkc")
    assert assert_same(emul, norm, ["Ａ́", "①́", "ｆ́x", "ｆ̈́ ｆ‍ ｆि", "\r\n", "A\r\nA"], 16) == []


def test_long_words_go_to_the_host(emul):
    """a text whose kept words include one longer than AC_UNIGRAM_MAX_WORD bytes ('▁' counted) is left to the host; words of
    exactly that many bytes, and long words past the kept ones, stay on the device; the composed rows equal the library's"""
    from adaptive_classifier_b200.tokenizer import UNIGRAM_MAX_WORD as M
    tok = uc.make_unigram()
    texts = ["x " + "a" * (M - 3), "x " + "a" * (M - 2), "日" * ((M - 3) // 3), "日" * ((M - 3) // 3 + 1), "a" * 1_000_000,
             "ok " * 20 + "a" * 50000, "short text"]
    ref = tok(texts, max_length=16, truncation=True)["input_ids"]
    tokens, lengths, max_len, _, _ = run_emul(emul, _spec(tok), texts, 16)
    left = [i for i in range(len(texts)) if lengths[i] < 0]
    assert left == [1, 3, 4]
    assert all(tokens[i, : lengths[i]].tolist() == ref[i] for i in range(len(texts)) if i not in left)


def test_kernels_under_address_sanitizer(monkeypatch):
    """a 1 MB word, 8192-token rows, words of AC_UNIGRAM_MAX_WORD and one more byte, the longest expansions, and cut UTF-8,
    on a build with AddressSanitizer and a workspace of exactly the queried size"""
    from adaptive_classifier_b200.tokenizer import UNIGRAM_MAX_WORD as M
    exe = _build("-fsanitize=address", "-fno-omit-frame-pointer")
    monkeypatch.setenv("ASAN_OPTIONS", "detect_leaks=0")
    tok = uc.make_unigram()
    texts = ["a" * 1_000_000, " ".join(uc.random_texts(300, seed=5)), "a" * (M - 1), "a" * M, "ﷺ" * 3000, "ﷺ " * 3000,
             "x" * (M - 2)] + uc.UNIGRAM_TRAPS
    assert_same(exe, tok, texts, 8192)
    run_emul(exe, _spec(tok), [b"x \xe4\xb8", b"\xf0\x9f", b"\xe4", b"\xef\xb7"], 8)
    run_emul(exe, _spec(tok), [b"x \xe4\xb8", b"\xf0\x9f", b"\xe4", b"\xef\xb7"], 8, mode=1)


def test_xlmr_tokenizers_are_accepted():
    from adaptive_classifier_b200.tokenizer import bpe_spec, unigram_spec, wordpiece_spec
    for tok in (uc.make_unigram(), uc.make_handmade([("▁a", -1.0)])):
        spec, why = unigram_spec(tok)
        assert spec is not None, why
        assert (spec["cls_id"], spec["sep_id"], spec["pad_id"], spec["unk_id"]) == (0, 2, 1, 3) and not spec["type_ids"]
        assert wordpiece_spec(tok)[0] is None and bpe_spec(tok)[0] is None
    assert unigram_spec(uc.make_unigram())[0]["grow"] == 11            # U+FDFA: 3 bytes to 33
    assert unigram_spec(uc.make_handmade([("▁a", -1.0)]))[0]["charsmap"] == []


def _with(edit):
    from tokenizers import Tokenizer
    from transformers import PreTrainedTokenizerFast
    tok = uc.make_handmade([("▁a", -1.0)], rule="nmt_nfkc")
    j = json.loads(tok.backend_tokenizer.to_str())
    edit(j)
    return PreTrainedTokenizerFast(tokenizer_object=Tokenizer.from_str(json.dumps(j)), bos_token="<s>", eos_token="</s>",
                                   cls_token="<s>", sep_token="</s>", pad_token="<pad>", unk_token="<unk>",
                                   mask_token="<mask>", model_input_names=["input_ids", "attention_mask"])


def _refused(tok, fragment):
    from adaptive_classifier_b200.tokenizer import unigram_spec
    spec, why = unigram_spec(tok)
    assert spec is None and fragment in why, why


def test_other_tokenizers_are_refused_with_a_reason():
    import bpe_corpus as bc
    import tokenizer_corpus as tc
    from tokenizers import AddedToken, normalizers
    _refused(tc.make_tokenizer("bert"), "is not Unigram")
    _refused(bc.make_bpe("roberta"), "is not Unigram")
    assert _spec(_with(lambda j: None))
    deberta = [{"type": "Replace", "pattern": {"Regex": r"\s{2,}|[\n\r\t]"}, "content": " "}, {"type": "NFC"},
               {"type": "Strip", "strip_left": True, "strip_right": True}]
    _refused(_with(lambda j: j.update(normalizer={"type": "Sequence", "normalizers": deberta})), "not Precompiled")
    albert = [{"type": "NFKD"}, {"type": "StripAccents"}, {"type": "Lowercase"}]
    _refused(_with(lambda j: j.update(normalizer={"type": "Sequence", "normalizers": albert})), "not Precompiled")
    _refused(_with(lambda j: j.update(normalizer={"type": "NFC"})), "not Precompiled")
    _refused(_with(lambda j: j["model"].update(byte_fallback=True)), "byte_fallback")
    _refused(_with(lambda j: j["model"].update(unk_id=None)), "unk_id")
    _refused(_with(lambda j: j.update(pre_tokenizer={"type": "Metaspace", "replacement": "▁", "prepend_scheme": "always",
                                                     "split": True})), "pre_tokenizer")
    _refused(_with(lambda j: j["pre_tokenizer"].update(pretokenizers=[{"type": "WhitespaceSplit"}, {
        "type": "Metaspace", "replacement": "▁", "prepend_scheme": "first", "split": True}])), "Metaspace is not")
    _refused(_with(lambda j: j["pre_tokenizer"].update(pretokenizers=[{"type": "WhitespaceSplit"}, {
        "type": "Metaspace", "replacement": "▁", "prepend_scheme": "always", "split": False}])), "Metaspace is not")
    copyright_key = uc.make_handmade([("▁a", -1.0)], rule=None)
    copyright_key.backend_tokenizer.normalizer = normalizers.Precompiled(uc.charsmap_from_rules({"©": "(c)"}))
    _refused(copyright_key, "starts with \u00a9 or \u00ae")
    _refused(_with(lambda j: j.update(post_processor={"type": "ByteLevel", "add_prefix_space": True, "trim_offsets": True, "use_regex": True})), "post_processor 'ByteLevel'")
    t = uc.make_unigram()
    t.add_tokens([AddedToken("foo", single_word=True)])
    _refused(t, "single_word=True")
    t = uc.make_unigram()
    t.truncation_side = "left"
    _refused(t, "left")
    t = uc.make_unigram()
    t.backend_tokenizer.encode_special_tokens = True
    _refused(t, "encode_special_tokens")
