"""Which Hugging Face tokenizers the device tokenizers (csrc/tokenizer.cu: WordPiece, byte-level BPE, Unigram) reproduce, and the Unicode
tables they run on.

The tables are derived by probing the installed `tokenizers` library (`normalize_str`, `pre_tokenize_str`), not from Python's
`unicodedata`: the Rust crates behind `tokenizers` carry their own Unicode version, and what must match is the library the host
path runs.  Needs no GPU.
"""
from __future__ import annotations

import hashlib
import json
import logging
import os
import tempfile
import unicodedata
from typing import Optional, Tuple

import numpy as np

logger = logging.getLogger(__name__)

N_CODEPOINTS = 0x110000
IDENTITY, BLOCKER = 0x80000000, 0x40000000
OTHER, SPACE, PUNCT = 0, 1, 2
_SEP = "#"            # probe separator: a starter every BertNormalizer flag combination keeps, and no other expansion holds
_ORDER_A, _ORDER_B = "\U0001D16D", "\U0001D165"   # non-spacing-mark-free combining marks, combining class 226 > 216

_CACHE = {}


def probe_codepoints() -> np.ndarray:
    return np.concatenate([np.arange(0xD800), np.arange(0xE000, N_CODEPOINTS)])


def pretokenizer_classes() -> np.ndarray:
    """uint8 [N_CODEPOINTS]: the class BertPreTokenizer gives each codepoint (SPACE: split and dropped, PUNCT: a word of its
    own, OTHER: part of a word).  Probed as one string of every codepoint: whitespace leaves its position uncovered by every
    piece, and the one-char pieces (punctuation, or a word char between two splits) are probed again between letters."""
    key = ("pre",)
    if key in _CACHE:
        return _CACHE[key]
    from tokenizers import pre_tokenizers
    pt = pre_tokenizers.BertPreTokenizer()
    cps = probe_codepoints()
    chars = list(map(chr, cps.tolist()))
    covered = np.zeros(len(chars), dtype=np.uint8)
    single = []
    for _, (a, b) in pt.pre_tokenize_str("".join(chars)):
        covered[a:b] = 1
        if b - a == 1:
            single.append(a)
    for _, (a, b) in pt.pre_tokenize_str("a" + "a".join(chars[i] for i in single) + "a"):
        if b - a == 1 and a % 2 == 1:
            covered[single[a // 2]] = 2
    cls = np.zeros(N_CODEPOINTS, dtype=np.uint8)
    cls[cps] = np.where(covered == 0, SPACE, np.where(covered == 2, PUNCT, OTHER))
    _CACHE[key] = cls
    return cls


def _normalize_each(normalizer, chars) -> list:
    """normalizer.normalize_str of every string of `chars` on its own, in one library call"""
    seps = [i for i, c in enumerate(chars) if _SEP in c]
    rest = [c for c in chars if _SEP not in c]
    out = normalizer.normalize_str(_SEP + _SEP.join(rest) + _SEP).split(_SEP)
    assert len(out) == len(rest) + 2, "probe separator split"
    out = out[1:-1]
    for i in seps:
        out.insert(i, normalizer.normalize_str(chars[i]))
    return out


def _reorder_ranks(nz, marks) -> dict:
    """{mark: rank} for the codepoints of `marks` the library reorders against another one: the ranks 1, 2, ... order them
    as the library's combining classes do, read from how many marks each one moves behind.  A candidate it never reorders against any other, in either
    direction, is a starter to it and is left out (rank 0)."""
    n = len(marks)
    if n < 2:
        return {}
    pairs = [chr(a) + chr(b) for a in marks for b in marks]
    swapped = np.array([o == p[::-1] != p for o, p in zip(_normalize_each(nz, pairs), pairs)], dtype=bool).reshape(n, n)
    moved = swapped.any(axis=1) | swapped.any(axis=0)
    below = swapped.sum(axis=1)                     # monotone in the class: equal classes move behind the same marks
    dense = {v: r + 1 for r, v in enumerate(sorted(set(below[moved].tolist())))}
    return {a: dense[int(below[i])] for i, a in enumerate(marks) if moved[i]}


def _disk_cache_path(key, kind: str = "wordpiece") -> str:
    """file of the tables for `key` under the user's cache directory; the name carries the tokenizers version, the flags and a
    hash of this module, so a changed library or a changed probe never reads an old file"""
    with open(__file__, "rb") as f:
        src = hashlib.sha256(f.read()).hexdigest()[:16]
    root = os.environ.get("XDG_CACHE_HOME") or os.path.join(os.path.expanduser("~"), ".cache")
    name = f"{kind}-tables-" + "-".join(str(k) for k in key) + f"-{src}.npz"
    return os.path.join(root, "adaptive_classifier_b200", name)


def unicode_tables(clean_text: bool, handle_chinese_chars: bool, strip_accents: bool, lowercase: bool):
    """(norm uint32 [N_CODEPOINTS], cls uint8 [N_CODEPOINTS], pool uint32 [*]) in the layout of ac_tokenizer_spec, for the
    BertNormalizer with these flags (strip_accents resolved: None means lowercase).  Probing takes seconds, so the result is
    kept per flags in the process and, when the user's cache directory is writable, on disk."""
    import tokenizers
    key = (tokenizers.__version__, clean_text, handle_chinese_chars, strip_accents, lowercase)
    if key in _CACHE:
        return _CACHE[key]
    path = _disk_cache_path(key)
    try:
        with np.load(path) as z:
            res = (z["norm"], z["cls"], z["pool"])
    except (OSError, KeyError, ValueError):
        res = _probe_tables(*key[1:])
        try:
            os.makedirs(os.path.dirname(path), exist_ok=True)
            fd, tmp = tempfile.mkstemp(dir=os.path.dirname(path), suffix=".npz")
            with os.fdopen(fd, "wb") as f:
                np.savez(f, norm=res[0], cls=res[1], pool=res[2])
            os.replace(tmp, path)                      # whole files only: concurrent processes may build the same tables
        except OSError as e:
            logger.debug(f"tokenizer tables not cached on disk: {e}")
    _CACHE[key] = res
    return res


def _probe_tables(clean_text: bool, handle_chinese_chars: bool, strip_accents: bool, lowercase: bool):
    from tokenizers import normalizers
    nz = normalizers.BertNormalizer(clean_text=clean_text, handle_chinese_chars=handle_chinese_chars,
                                    strip_accents=strip_accents, lowercase=lowercase)
    cps = probe_codepoints()
    chars = list(map(chr, cps.tolist()))
    exp = _normalize_each(nz, chars)
    norm = np.zeros(N_CODEPOINTS, dtype=np.uint32)
    same = np.fromiter((e == c for e, c in zip(exp, chars)), dtype=bool, count=len(chars))
    norm[cps[same]] = IDENTITY
    pool, empty = [], []
    for c, e in zip(cps[~same].tolist(), [e for e, s in zip(exp, same) if not s]):
        if len(e) >= 32:
            raise ValueError(f"U+{c:04X} expands to {len(e)} codepoints")
        norm[c] = (len(pool) << 5) | len(e)
        pool.extend(map(ord, e))
        if not e:
            empty.append(c)
    cls = pretokenizer_classes().copy()
    if strip_accents:
        # canonical ordering: NFD sorts each run of marks by combining class before the non-spacing marks are removed.  The
        # classes are the library's (its Unicode version need not be Python's), read from how it orders pairs of surviving
        # codepoints; unicodedata only proposes the candidates
        survivors = set(cps[same].tolist())
        if any(unicodedata.combining(chr(c)) for c in set(pool) - survivors):
            raise ValueError("a mark that only occurs inside expansions cannot be ordered by probing")
        marks = sorted(c for c in survivors if unicodedata.combining(chr(c)))
        ranks = _reorder_ranks(nz, marks)
        if ranks:
            # codepoints Python does not know yet may be marks to the library: probe them against its lowest- and
            # highest-ranked marks (one of the two pairs reorders for any nonzero class)
            lo = min(ranks, key=ranks.get)
            hi = max(ranks, key=ranks.get)
            kept = cps[same]
            kept = kept[(kept < 0x40000) | ((kept >= 0xE0000) & (kept < 0xF0000))].tolist()
            new = [c for c in kept if unicodedata.category(chr(c)) == "Cn"]
            probes = _normalize_each(nz, [chr(hi) + chr(c) for c in new] + [chr(c) + chr(lo) for c in new])
            found = [c for i, c in enumerate(new) if probes[i] == chr(c) + chr(hi) or probes[len(new) + i] == chr(lo) + chr(c)]
            logger.debug(f"{len(found)} marks unknown to unicodedata")
            if found:
                ranks = _reorder_ranks(nz, sorted(set(marks) | set(found)))
        for a, rank in ranks.items():
            if rank > 63:
                raise ValueError("more than 63 canonical-ordering ranks")
            cls[a] |= rank << 2
        # a removed codepoint between two marks either lets them reorder (removed before NFD, or a mark of nonzero class)
        # or blocks them (a removed mark of class 0).  Control, format and private-use codepoints are removed by clean_text
        # before NFD runs, so only the others are probed
        empty = [c for c in empty if unicodedata.category(chr(c)) not in ("Cc", "Cf", "Co")] if clean_text else empty
        if empty and _normalize_each(nz, [_ORDER_A + _ORDER_B]) == [_ORDER_B + _ORDER_A]:
            probes = _normalize_each(nz, [_ORDER_A + chr(c) + _ORDER_B for c in empty])
            norm[[c for c, o in zip(empty, probes) if o != _ORDER_B + _ORDER_A]] |= BLOCKER
    return norm, cls, np.asarray(pool, dtype=np.uint32)


_REPRESENTATIVE = ["Hello World", "  déjà vu, NAÏVE café!  ", "中文字符 and 𠀀", "İstanbul ΣΟΦΟΣ", "a\tb\nc d　e",
                   "tab\x00null�", "emoji 👩‍👩‍👧 $5+<3>", "x" * 120]


def wordpiece_spec(tokenizer) -> Tuple[Optional[dict], str]:
    """(spec, "") when the tokenizer is one the device kernel reproduces id for id, else (None, reason).  The decision is read
    from `backend_tokenizer.to_str()`, the pipeline that actually runs, and accepts nothing looser than:
    WordPiece model, BertNormalizer, BertPreTokenizer, a single-sequence post-processor "[special] A [special]" with type id 0,
    right truncation and padding, added tokens with normalized = false and single_word = false, and a Python wrapper that
    passes the text through unchanged."""
    bt = getattr(tokenizer, "backend_tokenizer", None)
    if bt is None:
        return None, "no Rust `tokenizers` backend (slow tokenizer)"
    j = json.loads(bt.to_str())
    model, nrm, pre, post = j.get("model") or {}, j.get("normalizer") or {}, j.get("pre_tokenizer") or {}, j.get("post_processor") or {}
    if model.get("type") != "WordPiece":
        return None, f"model {model.get('type')!r} is not WordPiece"
    if nrm.get("type") != "BertNormalizer":
        return None, f"normalizer {nrm.get('type')!r} is not BertNormalizer"
    if pre.get("type") != "BertPreTokenizer":
        return None, f"pre_tokenizer {pre.get('type')!r} is not BertPreTokenizer"
    vocab = model["vocab"]
    pt = post.get("type")
    if pt == "TemplateProcessing":
        single = post.get("single") or []
        kinds = [next(iter(x)) for x in single]
        if kinds != ["SpecialToken", "Sequence", "SpecialToken"] or any(next(iter(x.values())).get("type_id", 0) for x in single):
            return None, "post-processor template is not '[special] A [special]' with type id 0"
        ids = []
        for x in (single[0], single[2]):
            st = post["special_tokens"].get(x["SpecialToken"]["id"], {})
            if len(st.get("ids", [])) != 1:
                return None, "post-processor special token with more than one id"
            ids.append(st["ids"][0])
        cls_id, sep_id = ids
    elif pt in ("BertProcessing", "RobertaProcessing"):
        cls_id, sep_id = post["cls"][1], post["sep"][1]
    else:
        return None, f"post_processor {pt!r} is not TemplateProcessing / BertProcessing / RobertaProcessing"
    if getattr(tokenizer, "truncation_side", "right") != "right" or getattr(tokenizer, "padding_side", "right") != "right":
        return None, "left truncation or left padding"
    added = j.get("added_tokens") or []
    for a in added:
        if a.get("normalized", True) or a.get("single_word", False):
            return None, f"added token {a.get('content')!r} with normalized={a.get('normalized')} single_word={a.get('single_word')}"
    if "" in vocab:
        return None, "the vocab has an empty entry"
    unk = model.get("unk_token")
    if unk not in vocab:
        return None, f"unk_token {unk!r} is not in the vocab"
    prefix = model.get("continuing_subword_prefix", "##").encode("utf-8")
    if len(prefix) > 16:
        return None, "continuing_subword_prefix longer than 16 bytes"
    if tokenizer.pad_token_id is None:
        return None, "no pad token"
    try:
        # the transformers wrapper must hand the text to the backend unchanged
        wrapped = tokenizer(_REPRESENTATIVE)["input_ids"]
        backend = [e.ids for e in bt.encode_batch(_REPRESENTATIVE)]
    except Exception as e:                       # noqa: BLE001 -- any failure means: not a shape we reproduce
        return None, f"probe encoding failed: {e}"
    if wrapped != backend:
        return None, "the Python wrapper changes the text before the backend sees it"
    strip = nrm.get("strip_accents")
    lower = bool(nrm.get("lowercase", True))
    spec = dict(vocab=vocab, added=[(a["content"], a["id"]) for a in added], prefix=prefix,
                cls_id=int(cls_id), sep_id=int(sep_id), pad_id=int(tokenizer.pad_token_id), unk_id=int(vocab[unk]),
                max_input_chars=int(model.get("max_input_chars_per_word", 100)),
                flags=(bool(nrm.get("clean_text", True)), bool(nrm.get("handle_chinese_chars", True)),
                       lower if strip is None else bool(strip), lower),
                type_ids="token_type_ids" in getattr(tokenizer, "model_input_names", ()))
    return spec, ""


# ================================================================ byte-level BPE (csrc/tokenizer.cu, tokenize_bpe_*)
BPE_L, BPE_N, BPE_S, BPE_RUST = 1, 2, 4, 8
FOLD_LETTERS = "strevmld"                   # class bits 4-7: 1 + the index of the letter a codepoint matches under (?i)
SPLIT_GPT2, SPLIT_LLAMA3 = 0, 1
LLAMA3_PATTERN = (r"(?i:'s|'t|'re|'ve|'m|'ll|'d)|[^\r\n\p{L}\p{N}]?\p{L}+|\p{N}{1,3}| ?[^\s\p{L}\p{N}]+[\r\n]*|\s*[\r\n]+"
                  r"|\s+(?!\S)|\s+")
MAX_WORD = 1024                             # AC_BPE_MAX_WORD


def _uncovered(pre_tokenizer, chars) -> np.ndarray:
    """bool per char of `chars`: no piece of pre_tokenize_str covers it (what a 'removed' split or a whitespace split drops)"""
    covered = np.zeros(len(chars), dtype=bool)
    for _, (a, b) in pre_tokenizer.pre_tokenize_str("".join(chars)):
        covered[a:b] = True
    return ~covered


def bpe_classes() -> np.ndarray:
    """uint8 [N_CODEPOINTS] in the layout of ac_bpe_tokenizer_spec.cls: \\p{L}, \\p{N} and \\s as the library's regex engine
    (Oniguruma) matches them, Rust's char::is_whitespace (which lstrip / rstrip strip), and the letter of s t r e v m l d a
    codepoint matches case-insensitively.  Each class is one library call over every codepoint: a 'removed' split of a
    one-char pattern drops exactly the codepoints it matches, WhitespaceSplit the whitespace.  Kept in the process and on disk."""
    import tokenizers
    key = ("bpe", tokenizers.__version__)
    if key in _CACHE:
        return _CACHE[key]
    path = _disk_cache_path(key[1:], "bpe")
    try:
        with np.load(path) as z:
            cls = z["cls"]
    except (OSError, KeyError, ValueError):
        from tokenizers import Regex, pre_tokenizers
        cps = probe_codepoints()
        chars = list(map(chr, cps.tolist()))
        sub = np.zeros(len(chars), dtype=np.uint8)
        for bit, pat in ((BPE_L, r"\p{L}"), (BPE_N, r"\p{N}"), (BPE_S, r"\s")):
            sub |= np.where(_uncovered(pre_tokenizers.Split(Regex(pat), "removed"), chars), bit, 0).astype(np.uint8)
        sub |= np.where(_uncovered(pre_tokenizers.WhitespaceSplit(), chars), BPE_RUST, 0).astype(np.uint8)
        for i, letter in enumerate(FOLD_LETTERS):
            hit = _uncovered(pre_tokenizers.Split(Regex(f"(?i:{letter})"), "removed"), chars)
            if (sub[hit] >> 4).any():
                raise ValueError(f"a codepoint matches two contraction letters under (?i) ({letter!r})")
            sub |= np.where(hit, (i + 1) << 4, 0).astype(np.uint8)
        cls = np.zeros(N_CODEPOINTS, dtype=np.uint8)
        cls[cps] = sub
        try:
            os.makedirs(os.path.dirname(path), exist_ok=True)
            fd, tmp = tempfile.mkstemp(dir=os.path.dirname(path), suffix=".npz")
            with os.fdopen(fd, "wb") as f:
                np.savez(f, cls=cls)
            os.replace(tmp, path)
        except OSError as e:
            logger.debug(f"tokenizer tables not cached on disk: {e}")
    _CACHE[key] = cls
    return cls


def byte_level_map() -> dict:
    """{byte-level symbol: byte}: GPT-2's bytes_to_unicode, which ByteLevel applies to every byte of a piece"""
    keep = list(range(ord("!"), ord("~") + 1)) + list(range(ord("¡"), ord("¬") + 1)) + list(range(ord("®"), ord("ÿ") + 1))
    out, n = {}, 0
    for b in range(256):
        if b in keep:
            out[chr(b)] = b
        else:
            out[chr(256 + n)] = b
            n += 1
    return out


def _special_pair(post) -> Tuple[Optional[Tuple[int, int]], str]:
    """(cls id, sep id) of a single-sequence post-processor '[special] A [special]' with type id 0"""
    pt = post.get("type")
    if pt == "Sequence":
        procs = post.get("processors") or []
        rest = [p for p in procs if p.get("type") != "ByteLevel"]       # ByteLevel only moves offsets
        if len(rest) != 1 or rest[0].get("type") == "Sequence":
            return None, "post-processor Sequence is not ByteLevel and one '[special] A [special]' processor"
        return _special_pair(rest[0])
    if pt == "TemplateProcessing":
        single = post.get("single") or []
        kinds = [next(iter(x)) for x in single]
        if kinds != ["SpecialToken", "Sequence", "SpecialToken"] or any(next(iter(x.values())).get("type_id", 0) for x in single):
            return None, "post-processor template is not '[special] A [special]' with type id 0"
        ids = []
        for x in (single[0], single[2]):
            st = post["special_tokens"].get(x["SpecialToken"]["id"], {})
            if len(st.get("ids", [])) != 1:
                return None, "post-processor special token with more than one id"
            ids.append(st["ids"][0])
        return (int(ids[0]), int(ids[1])), ""
    if pt in ("BertProcessing", "RobertaProcessing"):
        return (int(post["cls"][1]), int(post["sep"][1])), ""
    return None, f"post_processor {pt!r} is not TemplateProcessing / BertProcessing / RobertaProcessing"


def _rust_space(ch: str) -> bool:
    return bool(bpe_classes()[ord(ch)] & BPE_RUST)


def _added_and_wrapper(tokenizer, bt, added) -> str:
    """"" when the truncation and padding sides, the added tokens and the Python wrapper are ones the BPE and Unigram split
    kernels reproduce (added tokens matched in two passes with lstrip / rstrip), else the reason"""
    if getattr(tokenizer, "truncation_side", "right") != "right" or getattr(tokenizer, "padding_side", "right") != "right":
        return "left truncation or left padding"
    if getattr(bt, "encode_special_tokens", False):
        return "encode_special_tokens splits the special tokens"
    for a in added:
        if a.get("single_word", False):
            return f"added token {a.get('content')!r} with single_word=True"
        if not a.get("content"):
            return "empty added token"
    for norm in (False, True):
        group = [a for a in added if bool(a.get("normalized", True)) == norm]
        if any(a.get("rstrip") for a in group) and any(_rust_space(a["content"][0]) for a in group):
            # the library resumes its scan inside the whitespace an rstrip token took, where such a token may match
            return "an rstrip added token next to one that starts with whitespace"
    if tokenizer.pad_token_id is None:
        return "no pad token"
    probe = _REPRESENTATIVE + [f"x{a['content']}y {a['content']} " for a in added]
    try:
        wrapped = tokenizer(probe)["input_ids"]
        backend = [e.ids for e in bt.encode_batch(probe)]
    except Exception as e:                       # noqa: BLE001 -- any failure means: not a shape we reproduce
        return f"probe encoding failed: {e}"
    if wrapped != backend:
        return "the Python wrapper changes the text before the backend sees it"
    return ""


def bpe_spec(tokenizer) -> Tuple[Optional[dict], str]:
    """(spec, "") when the tokenizer is a byte-level BPE tokenizer the device kernels reproduce id for id, else (None, reason).
    Read from `backend_tokenizer.to_str()`; accepts nothing looser than: a BPE model without dropout, affixes or byte fallback
    whose vocab holds all 256 byte symbols, no normalizer, ByteLevel(use_regex) or Split(Llama-3 pattern) + ByteLevel, a
    '[special] A [special]' post-processor with type id 0 (optionally in a Sequence with ByteLevel), right truncation and
    padding, added tokens with single_word = false, and a Python wrapper that passes the text through unchanged."""
    bt = getattr(tokenizer, "backend_tokenizer", None)
    if bt is None:
        return None, "no Rust `tokenizers` backend (slow tokenizer)"
    j = json.loads(bt.to_str())
    model, pre, post = j.get("model") or {}, j.get("pre_tokenizer") or {}, j.get("post_processor") or {}
    if model.get("type") != "BPE":
        return None, f"model {model.get('type')!r} is not BPE"
    if model.get("dropout") is not None:
        return None, "BPE dropout"
    if model.get("continuing_subword_prefix") or model.get("end_of_word_suffix"):
        return None, "BPE continuing_subword_prefix / end_of_word_suffix"
    if model.get("byte_fallback"):
        return None, "BPE byte_fallback"
    if j.get("normalizer") is not None:
        return None, f"normalizer {(j.get('normalizer') or {}).get('type')!r} (byte-level BPE takes none)"
    if pre.get("type") == "ByteLevel":
        if not pre.get("use_regex", True):
            return None, "ByteLevel pre-tokenizer without use_regex"
        split, prefix_space = SPLIT_GPT2, bool(pre.get("add_prefix_space", False))
    elif pre.get("type") == "Sequence":
        seq = pre.get("pretokenizers") or []
        if len(seq) != 2 or seq[0].get("type") != "Split" or seq[1].get("type") != "ByteLevel":
            return None, "pre_tokenizer Sequence is not [Split, ByteLevel]"
        sp, bl = seq
        if (sp.get("pattern") or {}).get("Regex") != LLAMA3_PATTERN:
            return None, f"Split pattern {sp.get('pattern')!r} is not the Llama-3 pattern"
        if sp.get("behavior") != "Isolated" or sp.get("invert"):
            return None, "Split is not Isolated without invert"
        if bl.get("use_regex", True) or bl.get("add_prefix_space", False):
            return None, "ByteLevel after Split with use_regex or add_prefix_space"
        split, prefix_space = SPLIT_LLAMA3, False
    else:
        return None, f"pre_tokenizer {pre.get('type')!r} is not ByteLevel or [Split, ByteLevel]"
    vocab = model["vocab"]
    sym = byte_level_map()
    if any(s not in vocab for s in sym):
        return None, "the vocab lacks some of the 256 byte-level symbols"
    pair, why = _special_pair(post)
    if pair is None:
        return None, why
    added = j.get("added_tokens") or []
    why = _added_and_wrapper(tokenizer, bt, added)
    if why:
        return None, why
    merges = []
    for m in model.get("merges") or []:
        a, b = m.split(" ", 1) if isinstance(m, str) else m
        merges.append((vocab[a], vocab[b], vocab[a + b]))
    spec = dict(split=split, prefix_space=prefix_space, ignore_merges=bool(model.get("ignore_merges", False)),
                vocab=vocab, byte_ids=[vocab[s] for s in sorted(sym, key=sym.get)], merges=merges,
                added=[(a["content"], int(a["id"]), bool(a.get("normalized", True)), bool(a.get("lstrip", False)),
                        bool(a.get("rstrip", False))) for a in added],
                cls_id=pair[0], sep_id=pair[1], pad_id=int(tokenizer.pad_token_id),
                type_ids="token_type_ids" in getattr(tokenizer, "model_input_names", ()))
    return spec, ""


def bpe_vocab_bytes(vocab: dict) -> Tuple[list, list]:
    """(raw byte strings, ids) of the vocab entries made of byte-level symbols only, mapped back to the bytes they stand for"""
    sym = byte_level_map()
    words, ids = [], []
    for w, i in vocab.items():
        if all(c in sym for c in w):
            words.append(bytes(sym[c] for c in w))
            ids.append(int(i))
    return words, ids


def pack_strings(strings) -> Tuple[np.ndarray, np.ndarray]:
    """UTF-8 bytes of the strings back to back, and int64 offsets [n + 1]"""
    enc = [s.encode("utf-8") for s in strings]
    off = np.zeros(len(enc) + 1, dtype=np.int64)
    np.cumsum([len(e) for e in enc], out=off[1:])
    return np.frombuffer(b"".join(enc) or b"\0", dtype=np.uint8), off


# ================================================================ SentencePiece Unigram, XLM-R shape (csrc/tokenizer.cu, tokenize_unigram_*)
G_JOIN, G_CONTROL, G_PREPEND = 1, 2, 4      # grapheme class bits; BPE_RUST (8) is Rust whitespace, as in bpe_classes
METASPACE = "▁"
# the Extended_Pictographic chars shorter than 3 bytes: "©" + ZWJ is a 5-byte prefix of a longer emoji ZWJ cluster (GB11),
# which the device does not model, so it reads "©‍©" as "©‍" + "©"; that differs from the library only when a charsmap key
# starts with one of them (none of sentencepiece's built-in rules has such a key)
_EXT_PICT_2BYTE = ("©".encode(), "®".encode())
UNIGRAM_MAX_WORD = 4096                     # AC_UNIGRAM_MAX_WORD


def decode_charsmap(blob: bytes) -> list:
    """[(key bytes, value bytes)] of a SentencePiece `precompiled_charsmap`: a 4-byte little-endian trie size, a double-array
    trie of uint32 units (darts-clone layout: bits 0-7 the label, bit 8 has-leaf, bit 9 scales the offset in bits 10-31; a
    leaf unit's bits 0-30 are the value) and the pool of NUL-terminated values the leaves point into.  Walked breadth first,
    every live node against every byte at once."""
    n = int.from_bytes(blob[:4], "little")
    if n % 4 or 4 + n > len(blob):
        raise ValueError("precompiled_charsmap: trie size past the blob")
    units = np.frombuffer(blob, dtype="<u4", count=n // 4, offset=4).astype(np.int64)
    pool = blob[4 + n:]
    if not len(units):
        return []

    def offset(u):
        return (u >> 10) << ((u & (1 << 9)) >> 6)

    labels = np.arange(1, 256, dtype=np.int64)
    pos = np.asarray([offset(units[0])], dtype=np.int64)
    keys = [b""]
    out = []
    for _ in range(64):                         # no key is longer; a deeper walk means a corrupt trie
        if not len(pos):
            break
        child = pos[:, None] ^ labels[None, :]
        inside = child < len(units)
        u = np.where(inside, units[np.where(inside, child, 0)], -1)
        hit = inside & ((u & ((1 << 31) | 0xFF)) == labels[None, :])
        pi, li = np.nonzero(hit)
        ch, uu = child[pi, li], u[pi, li]
        nxt = ch ^ offset(uu)
        if (nxt >= len(units)).any():
            raise ValueError("precompiled_charsmap: node past the trie")
        new_keys = [keys[p] + bytes([int(labels[l])]) for p, l in zip(pi.tolist(), li.tolist())]
        for k, leaf, q in zip(new_keys, ((uu >> 8) & 1).tolist(), nxt.tolist()):
            if leaf:
                v = int(units[q] & 0x7FFFFFFF)
                end = pool.find(b"\0", v)
                if v > len(pool) or end < 0:
                    raise ValueError("precompiled_charsmap: value past the pool")
                out.append((k, bytes(pool[v:end])))
        pos, keys = nxt, new_keys
    else:
        raise ValueError("precompiled_charsmap: key longer than 64 bytes")
    return sorted(out)


def charsmap_tables(blob: bytes) -> dict:
    """decoded charsmap of a Precompiled normalizer: pairs, and the largest expansion in value bytes per key byte (rounded up,
    at least 1), which sizes the device workspace.  Every single-codepoint key is checked against the library's
    normalize_str: a blob this decoder misreads is refused rather than tokenized differently.  Kept per blob in the process."""
    key = ("charsmap", hashlib.sha256(blob).hexdigest())
    if key in _CACHE:
        return _CACHE[key]
    from tokenizers import normalizers
    pairs = decode_charsmap(blob)
    single = [(k.decode("utf-8"), v.decode("utf-8")) for k, v in pairs if len(k.decode("utf-8", "replace")) == 1]
    nz = normalizers.Precompiled(blob)
    bad = [k for k, v in single if nz.normalize_str(k) != v]
    if bad:
        raise ValueError(f"precompiled_charsmap decoded differently from the library for {len(bad)} keys, e.g. {bad[0]!r}")
    grow = max([1] + [-(-len(v) // len(k)) for k, v in pairs])
    res = dict(pairs=pairs, grow=grow)
    _CACHE[key] = res
    return res


def all_to_b_charsmap() -> bytes:
    """a charsmap that maps every codepoint but NUL and the surrogates to 'b' ('b' included), compiled by sentencepiece from a
    rule table: under it, normalize_str of a string shorter than 6 bytes has one char per grapheme cluster the library cuts
    it into (a cluster that holds NUL is NUL alone)"""
    import io
    import sentencepiece as spm
    from sentencepiece import sentencepiece_model_pb2
    with tempfile.TemporaryDirectory() as d:
        rules = os.path.join(d, "rules.tsv")
        with open(rules, "w") as f:
            f.writelines(f"{c:X}\t62\n" for c in probe_codepoints().tolist() if c)
        corpus = [f"probe line {i} of the grapheme class table" for i in range(200)]
        model = io.BytesIO()
        spm.SentencePieceTrainer.train(sentence_iterator=iter(corpus), model_writer=model, vocab_size=60, model_type="unigram",
                                       hard_vocab_limit=False, normalization_rule_tsv=rules, minloglevel=2)
    m = sentencepiece_model_pb2.ModelProto()
    m.ParseFromString(model.getvalue())
    return m.normalizer_spec.precompiled_charsmap


def unigram_classes() -> np.ndarray:
    """uint8 [N_CODEPOINTS] in the layout of ac_unigram_tokenizer_spec.cls: the grapheme cluster classes of the library's
    segmentation (unicode-segmentation) that can change a Precompiled result, and Rust whitespace (WhitespaceSplit, lstrip /
    rstrip).  Under a charsmap mapping every codepoint to 'b', one 'b' means one cluster:
      G_JOIN     'a' + c is one cluster (Extend, ZWJ, SpacingMark);
      G_CONTROL  c + U+0301 is two (Control, CR, LF: nothing joins them, and they join nothing);
      G_PREPEND  c + 'x' is one (Prepend).
    Clusters of 6 bytes or more are normalized char by char, so the rules that only build such clusters (Hangul, regional
    indicators, emoji ZWJ sequences, conjuncts) need no class; unigram_spec refuses the one charsmap shape where that would
    show (see _EXT_PICT_2BYTE).  The count of output chars, not which char comes out, decides each bit, so the mapping target
    is probed like any other codepoint.  Kept in the process and on disk."""
    import tokenizers
    key = ("unigram", tokenizers.__version__)
    if key in _CACHE:
        return _CACHE[key]
    path = _disk_cache_path(key[1:], "unigram")
    try:
        with np.load(path) as z:
            cls = z["cls"]
    except (OSError, KeyError, ValueError):
        from tokenizers import normalizers, pre_tokenizers
        nz = normalizers.Precompiled(all_to_b_charsmap())
        cps = probe_codepoints()
        chars = list(map(chr, cps.tolist()))

        def clusters(s):
            return len(nz.normalize_str(s))

        sub = np.zeros(len(chars), dtype=np.uint8)
        sub |= np.fromiter((clusters("a" + c) == 1 for c in chars), dtype=bool, count=len(chars)).astype(np.uint8) * G_JOIN
        sub |= np.fromiter((len(c.encode()) < 4 and clusters(c + "́") == 2 for c in chars), dtype=bool,
                           count=len(chars)).astype(np.uint8) * G_CONTROL
        sub |= np.fromiter((clusters(c + "x") == 1 for c in chars), dtype=bool, count=len(chars)).astype(np.uint8) * G_PREPEND
        sub |= np.where(_uncovered(pre_tokenizers.WhitespaceSplit(), chars), BPE_RUST, 0).astype(np.uint8)
        if clusters("\r\n") != 1:
            raise ValueError("CR LF is not one grapheme cluster to this library")
        cls = np.zeros(N_CODEPOINTS, dtype=np.uint8)
        cls[cps] = sub
        try:
            os.makedirs(os.path.dirname(path), exist_ok=True)
            fd, tmp = tempfile.mkstemp(dir=os.path.dirname(path), suffix=".npz")
            with os.fdopen(fd, "wb") as f:
                np.savez(f, cls=cls)
            os.replace(tmp, path)
        except OSError as e:
            logger.debug(f"tokenizer tables not cached on disk: {e}")
    _CACHE[key] = cls
    return cls


def unigram_spec(tokenizer) -> Tuple[Optional[dict], str]:
    """(spec, "") when the tokenizer is a SentencePiece Unigram tokenizer of the XLM-RoBERTa shape that the device kernels
    reproduce id for id, else (None, reason).  Read from `backend_tokenizer.to_str()` (what AutoTokenizer actually runs);
    accepts nothing looser than: a Unigram model without byte_fallback and with an unk_id, no normalizer or Precompiled, the
    pre-tokenizer Sequence[WhitespaceSplit, Metaspace('▁', prepend_scheme 'always', split)], a '[special] A [special]'
    post-processor with type id 0, right truncation and padding, added tokens with single_word = false, and a Python wrapper
    that passes the text through unchanged."""
    import base64
    bt = getattr(tokenizer, "backend_tokenizer", None)
    if bt is None:
        return None, "no Rust `tokenizers` backend (slow tokenizer)"
    j = json.loads(bt.to_str())
    model, nrm, pre, post = j.get("model") or {}, j.get("normalizer"), j.get("pre_tokenizer") or {}, j.get("post_processor") or {}
    if model.get("type") != "Unigram":
        return None, f"model {model.get('type')!r} is not Unigram"
    if model.get("byte_fallback"):
        return None, "Unigram byte_fallback"
    if model.get("unk_id") is None:
        return None, "Unigram without unk_id"
    if nrm is not None and nrm.get("type") != "Precompiled":
        return None, f"normalizer {nrm.get('type')!r} is not Precompiled (or none)"
    seq = pre.get("pretokenizers") or []
    if pre.get("type") != "Sequence" or [p.get("type") for p in seq] != ["WhitespaceSplit", "Metaspace"]:
        return None, f"pre_tokenizer {pre.get('type')!r} is not Sequence[WhitespaceSplit, Metaspace]"
    ms = seq[1]
    if ms.get("replacement") != METASPACE or ms.get("prepend_scheme") != "always" or not ms.get("split", True):
        return None, "Metaspace is not ('▁', prepend_scheme 'always', split)"
    pair, why = _special_pair(post)
    if pair is None:
        return None, why
    vocab = model.get("vocab") or []
    if not vocab or any(not p for p, _ in vocab):
        return None, "empty Unigram vocab or an empty piece"
    unk_id = int(model["unk_id"])
    if not 0 <= unk_id < len(vocab):
        return None, "unk_id outside the vocab"
    added = j.get("added_tokens") or []
    why = _added_and_wrapper(tokenizer, bt, added)
    if why:
        return None, why
    try:
        cmap = charsmap_tables(base64.b64decode(nrm["precompiled_charsmap"])) if nrm else dict(pairs=[], grow=1)
    except (ValueError, KeyError, TypeError) as e:
        return None, f"precompiled_charsmap: {e}"
    if any(k.startswith(_EXT_PICT_2BYTE) for k, _ in cmap["pairs"]):
        return None, "a charsmap key starts with \u00a9 or \u00ae, where emoji ZWJ sequences would change its clusters"
    try:
        unigram_classes()
    except ImportError as e:
        return None, f"the grapheme class table is probed through sentencepiece, which is not installed ({e})"
    spec = dict(pieces=[(p.encode("utf-8"), float(s)) for p, s in vocab], unk_id=unk_id, charsmap=cmap["pairs"],
                grow=cmap["grow"],
                added=[(a["content"], int(a["id"]), bool(a.get("normalized", True)), bool(a.get("lstrip", False)),
                        bool(a.get("rstrip", False))) for a in added],
                cls_id=pair[0], sep_id=pair[1], pad_id=int(tokenizer.pad_token_id),
                type_ids="token_type_ids" in getattr(tokenizer, "model_input_names", ()))
    return spec, ""
