// tokenizer.cu -- WordPiece tokenization on the device for BERT-family tokenizers (BertNormalizer + BertPreTokenizer +
// WordPiece + "[special] A [special]"), ids identical to the Hugging Face `tokenizers` pipeline (adaptive_classifier_b200/
// tokenizer.py decides which tokenizers qualify and builds the Unicode tables by probing the installed library).
//
// One thread per text walks its UTF-8 bytes once: added tokens (normalized = false) are matched on the raw bytes, every other
// codepoint is replaced by its normalized expansion (table), the expansion's codepoints are split into words by their
// pre-tokenizer class (table), and each finished word is cut by greedy longest-match WordPiece against an open-addressing hash
// table of the vocab.  The walk stops once max_length - 2 tokens exist: later words cannot change the kept ids.
//
// Byte-level BPE tokenizers (RoBERTa, ModernBERT, EuroBERT) run on three kernels further down, sharing the UTF-8 decoding,
// the handle, the uploads and tokenize_pack_kernel with WordPiece; SentencePiece Unigram tokenizers of the XLM-RoBERTa shape
// run on two kernels of their own and BPE's added-token trie and gather kernel.
//
// The file is plain SIMT C++: with AC_CPU_SHIM defined (tests/cpu_shim) only the kernels and the host-side table builder are
// compiled, so the control flow runs on the CPU as well.
#ifndef AC_CPU_SHIM
#include "common.cuh"
#endif
#include <algorithm>
#include <cstdint>
#include <cstring>
#include <vector>

namespace ac {
namespace tok {

constexpr int kCodepoints = 0x110000;
// norm[c]: kIdentity -> c maps to itself; else (offset << 5) | length into the pool, and kBlocker on an empty expansion that
// stops canonical reordering across it (a removed mark of combining class 0, e.g. U+034F)
constexpr uint32_t kIdentity = 0x80000000u, kBlocker = 0x40000000u, kOffsetMask = 0x3fffffffu;
// cls[c]: bits 0-1 the pre-tokenizer class of c as a normalized char, bits 2-7 its canonical-ordering rank (0: a starter)
enum { kOther = 0, kSpace = 1, kPunct = 2 };
constexpr int kMaxPrefix = 16;
constexpr uint32_t kFnvBasis = 2166136261u;

struct Tables {
    const uint32_t *norm;
    const uint8_t *cls;
    const uint32_t *pool;
    const int4 *slots;          // (id, hash, byte offset, byte length); id < 0: empty
    uint32_t slot_mask;
    const uint8_t *vocab_bytes;
    const uint8_t *added_bytes; // added tokens, longest first
    const int64_t *added_off;
    const int32_t *added_id;
    int n_added;
    uint32_t first_byte[8];     // bit set: some added token starts with this byte
    uint8_t prefix[kMaxPrefix];
    int prefix_len;
    int max_key;                // longest vocab entry in bytes
    int cls_id, sep_id, pad_id, unk_id, max_chars;
};

__host__ __device__ inline uint32_t fnv1a(uint32_t h, const uint8_t *p, int n) {
    for (int i = 0; i < n; ++i) h = (h ^ p[i]) * 16777619u;
    return h;
}

__device__ inline int vocab_find(const Tables &t, const uint8_t *s, int n, bool cont) {
    uint32_t h = kFnvBasis;
    int total = n;
    if (cont) {
        h = fnv1a(h, t.prefix, t.prefix_len);
        total += t.prefix_len;
    }
    h = fnv1a(h, s, n);
    for (uint32_t i = h & t.slot_mask;; i = (i + 1) & t.slot_mask) {
        const int4 e = t.slots[i];
        if (e.x < 0) return -1;
        if (static_cast<uint32_t>(e.y) != h || e.w != total) continue;
        const uint8_t *v = t.vocab_bytes + e.z;
        bool eq = true;
        int k = 0;
        if (cont)
            for (; k < t.prefix_len && eq; ++k) eq = v[k] == t.prefix[k];
        for (int j = 0; j < n && eq; ++j) eq = v[k + j] == s[j];
        if (eq) return e.x;
    }
}

// Python's str.encode gives valid UTF-8; anything else through the C ABI (a stray continuation byte, a lead byte past 0xF4, a
// sequence cut by the end of the text, a value past U+10FFFF) is read as one U+FFFD per byte and never past `end`
__device__ inline int utf8_decode(const uint8_t *p, const uint8_t *end, uint32_t &c) {
    const uint32_t b = p[0];
    if (b < 0x80) { c = b; return 1; }
    const int n = b >= 0xF0 ? 4 : b >= 0xE0 ? 3 : b >= 0xC0 ? 2 : 0;
    c = 0xFFFD;
    if (n == 0 || b > 0xF4 || end - p < n) return 1;
    uint32_t v = b & (0x7F >> n);
    for (int i = 1; i < n; ++i) {
        if ((p[i] & 0xC0) != 0x80) return 1;
        v = (v << 6) | (p[i] & 0x3F);
    }
    if (v < 0x110000) c = v;
    return n;
}

__device__ inline int utf8_encode(uint32_t c, uint8_t *o) {      // c < 0x110000
    if (c < 0x80) { o[0] = static_cast<uint8_t>(c); return 1; }
    if (c < 0x800) { o[0] = 0xC0 | (c >> 6); o[1] = 0x80 | (c & 0x3F); return 2; }
    if (c < 0x10000) { o[0] = 0xE0 | (c >> 12); o[1] = 0x80 | ((c >> 6) & 0x3F); o[2] = 0x80 | (c & 0x3F); return 3; }
    o[0] = 0xF0 | (c >> 18); o[1] = 0x80 | ((c >> 12) & 0x3F); o[2] = 0x80 | ((c >> 6) & 0x3F); o[3] = 0x80 | (c & 0x3F);
    return 4;
}

// the word being collected: its normalized codepoints (only the first max_chars + 1 are kept: a longer word is [UNK] whatever
// it holds), its length in chars, and where the run of marks that canonical ordering may still permute begins
struct Word {
    uint32_t *cp;
    uint8_t *bytes;
    int len, run;
};

struct Out {
    int32_t *ids;
    int n, limit;               // ids written; content tokens are written while n < limit = max_length - 1
};

// WordPiece (tokenizers' models/wordpiece): greedy longest match from the left, continuation pieces looked up as prefix + piece;
// a word with more than max_chars chars, or with a position no piece matches, is one [UNK]
__device__ inline void word_flush(const Tables &t, Word &w, Out &o) {
    if (w.len == 0) return;
    const int len = w.len;
    w.len = 0;
    w.run = 0;
    if (len > t.max_chars) {
        if (o.n < o.limit) o.ids[o.n++] = t.unk_id;
        return;
    }
    int nb = 0;
    for (int i = 0; i < len; ++i) nb += utf8_encode(w.cp[i], w.bytes + nb);
    const int first = o.n;
    for (int start = 0; start < nb;) {
        const bool cont = start > 0;
        const int longest = t.max_key - (cont ? t.prefix_len : 0);
        int end = nb;
        if (end - start > longest) {               // no vocab entry is longer: start below it, on a char boundary
            end = start + (longest > 0 ? longest : 0);
            while (end > start && (w.bytes[end] & 0xC0) == 0x80) --end;
        }
        int id = -1;
        while (end > start) {
            id = vocab_find(t, w.bytes + start, end - start, cont);
            if (id >= 0) break;
            do --end; while (end > start && (w.bytes[end] & 0xC0) == 0x80);
        }
        if (id < 0) {
            o.n = first;
            if (o.n < o.limit) o.ids[o.n++] = t.unk_id;
            return;
        }
        if (o.n < o.limit) o.ids[o.n] = id;
        ++o.n;                                     // counted past the limit too, so that an [UNK] verdict resets to `first`
        start = end;
    }
    if (o.n > o.limit) o.n = o.limit;
}

// append one normalized codepoint; a mark of nonzero rank moves in front of the marks of higher rank since the last starter
// (the stable canonical ordering of NFD, which the library applies before removing the nonspacing marks)
__device__ inline void word_push(const Tables &t, Word &w, uint32_t c) {
    const int r = t.cls[c] >> 2;
    if (w.len <= t.max_chars) {
        int j = w.len;
        if (r)
            for (; j > w.run && (t.cls[w.cp[j - 1]] >> 2) > r; --j) w.cp[j] = w.cp[j - 1];
        w.cp[j] = c;
    }
    ++w.len;
    if (!r) w.run = w.len;
}

__device__ inline void emit_codepoint(const Tables &t, Word &w, Out &o, uint32_t c) {
    const int k = t.cls[c] & 3;
    if (k == kOther) {
        word_push(t, w, c);
        return;
    }
    word_flush(t, w, o);                           // whitespace ends the word and is dropped; punctuation is a word of its own
    if (k == kPunct) {
        word_push(t, w, c);
        word_flush(t, w, o);
    }
}

// longest added token at p (the library's leftmost-longest match on the raw text), or -1
__device__ inline int match_added(const Tables &t, const uint8_t *p, const uint8_t *end) {
    for (int a = 0; a < t.n_added; ++a) {
        const int64_t o0 = t.added_off[a], n = t.added_off[a + 1] - o0;
        if (n > end - p) continue;
        bool eq = true;
        for (int64_t j = 0; j < n && eq; ++j) eq = t.added_bytes[o0 + j] == p[j];
        if (eq) return a;
    }
    return -1;
}

// tokens[b, 0 .. lengths[b]) = [CLS] pieces [SEP] of text b, truncated to max_length; *max_len = max over the batch (zeroed by
// the caller).  ws_cp / ws_bytes: (max_chars + 1) codepoints and 4 (max_chars + 1) bytes per text.
__global__ void __launch_bounds__(128) tokenize_wordpiece_kernel(Tables t, const uint8_t *text, const int64_t *offsets, int B,
                                                                 int max_length, int32_t *tokens, int32_t *lengths,
                                                                 int32_t *max_len, uint32_t *ws_cp, uint8_t *ws_bytes) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    const uint8_t *p = text + offsets[b], *end = text + offsets[b + 1];
    Out o{tokens + static_cast<int64_t>(b) * max_length, 0, max_length - 1};
    Word w{ws_cp + static_cast<int64_t>(b) * (t.max_chars + 1), ws_bytes + static_cast<int64_t>(b) * 4 * (t.max_chars + 1), 0, 0};
    o.ids[o.n++] = t.cls_id;
    while (p < end && o.n < o.limit) {
        if ((t.first_byte[*p >> 5] >> (*p & 31)) & 1u) {
            // lstrip / rstrip only widen the match over whitespace, which BertPreTokenizer drops anyway
            const int a = match_added(t, p, end);
            if (a >= 0) {
                word_flush(t, w, o);
                if (o.n < o.limit) o.ids[o.n++] = t.added_id[a];
                p += t.added_off[a + 1] - t.added_off[a];
                continue;
            }
        }
        uint32_t c;
        p += utf8_decode(p, end, c);
        const uint32_t e = t.norm[c];
        if (e & kIdentity) {
            emit_codepoint(t, w, o, c);
        } else if ((e & 31) == 0) {
            if (e & kBlocker) w.run = w.len;
        } else {
            const uint32_t *x = t.pool + ((e & kOffsetMask) >> 5);
            for (uint32_t i = 0; i < (e & 31); ++i) emit_codepoint(t, w, o, x[i]);
        }
    }
    word_flush(t, w, o);
    o.ids[o.n++] = t.sep_id;
    lengths[b] = o.n;
    atomicMax(max_len, o.n);
}

// ids / mask / type_ids [B, S]: the first lengths[b] tokens of row b, then pad_id with mask 0 (right padding, type id 0)
__global__ void tokenize_pack_kernel(const int32_t *tokens, const int32_t *lengths, int B, int max_length, int S, int pad_id,
                                     int32_t *ids, int32_t *mask, int32_t *type_ids) {
    const int64_t total = static_cast<int64_t>(B) * S;
    for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total;
         i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        const int64_t b = i / S, s = i - b * S;
        const bool v = s < lengths[b];
        ids[i] = v ? tokens[b * max_length + s] : pad_id;
        mask[i] = v ? 1 : 0;
        if (type_ids) type_ids[i] = 0;
    }
}

// ---------------------------------------------------------------- host side: the tables in the layout the kernel reads
struct HostTables {
    std::vector<int4> slots;
    std::vector<uint8_t> added_bytes;
    std::vector<int64_t> added_off;
    std::vector<int32_t> added_id;
    Tables t{};                     // scalars, prefix and first_byte filled; pointers left to the owner
};

// the open-addressing table (id, FNV-1a hash, byte offset, byte length) of n byte strings, load factor <= 1/2 so that every
// probe chain ends; returns nullptr, or what is wrong with the strings
inline const char *hash_byte_strings(const uint8_t *bytes, const int64_t *offsets, const int32_t *ids, int n,
                                     std::vector<int4> &slots, int &max_key) {
    size_t n_slots = 2;
    while (n_slots < 2 * static_cast<size_t>(n)) n_slots <<= 1;
    slots.assign(n_slots, int4{-1, 0, 0, 0});
    max_key = 0;
    for (int v = 0; v < n; ++v) {
        const int64_t o0 = offsets[v], len = offsets[v + 1] - o0;
        if (len <= 0 || o0 + len > INT32_MAX) return "empty vocab entry or vocab bytes over 2 GB";
        const uint32_t hash = fnv1a(kFnvBasis, bytes + o0, static_cast<int>(len));
        size_t i = hash & (n_slots - 1);
        while (slots[i].x >= 0) {
            const int4 &e = slots[i];
            if (e.w == len && !memcmp(bytes + e.z, bytes + o0, len)) return "duplicate vocab entry";
            i = (i + 1) & (n_slots - 1);
        }
        if (ids[v] < 0) return "negative vocab id";
        slots[i] = int4{ids[v], static_cast<int>(hash), static_cast<int>(o0), static_cast<int>(len)};
        max_key = std::max<int>(max_key, static_cast<int>(len));
    }
    return nullptr;
}

// returns nullptr, or what is wrong with the spec
inline const char *build_host_tables(const ac_tokenizer_spec &s, HostTables &h) {
    if (!s.norm || !s.cls || (s.pool_len && !s.pool) || !s.vocab_bytes || !s.vocab_offsets || !s.vocab_ids || s.n_vocab <= 0)
        return "null table or empty vocab";
    if (s.prefix_len < 0 || s.prefix_len > kMaxPrefix || (s.prefix_len && !s.prefix)) return "continuing_subword_prefix longer than 16 bytes";
    if (s.max_input_chars < 1) return "max_input_chars_per_word < 1";
    if (s.n_added < 0 || (s.n_added && (!s.added_bytes || !s.added_offsets || !s.added_ids))) return "bad added tokens";
    if (s.pool_len > (kOffsetMask >> 5)) return "expansion pool too large";
    int max_key = 0;
    if (const char *why = hash_byte_strings(s.vocab_bytes, s.vocab_offsets, s.vocab_ids, s.n_vocab, h.slots, max_key)) return why;
    const size_t n_slots = h.slots.size();
    std::vector<int> order(s.n_added);
    for (int a = 0; a < s.n_added; ++a) {
        order[a] = a;
        if (s.added_offsets[a + 1] <= s.added_offsets[a]) return "empty added token";
    }
    std::stable_sort(order.begin(), order.end(), [&](int x, int y) {
        return s.added_offsets[x + 1] - s.added_offsets[x] > s.added_offsets[y + 1] - s.added_offsets[y];
    });
    h.added_off.assign(1, 0);
    memset(h.t.first_byte, 0, sizeof(h.t.first_byte));
    for (int a : order) {
        const uint8_t *src = s.added_bytes + s.added_offsets[a];
        h.added_bytes.insert(h.added_bytes.end(), src, src + (s.added_offsets[a + 1] - s.added_offsets[a]));
        h.added_off.push_back(static_cast<int64_t>(h.added_bytes.size()));
        h.added_id.push_back(s.added_ids[a]);
        h.t.first_byte[src[0] >> 5] |= 1u << (src[0] & 31);
    }
    if (h.added_bytes.empty()) h.added_bytes.push_back(0);
    if (h.added_id.empty()) h.added_id.push_back(0);
    h.t.slot_mask = static_cast<uint32_t>(n_slots - 1);
    h.t.n_added = s.n_added;
    memcpy(h.t.prefix, s.prefix ? s.prefix : "", s.prefix_len);
    h.t.prefix_len = s.prefix_len;
    h.t.max_key = max_key;
    h.t.cls_id = s.cls_id;
    h.t.sep_id = s.sep_id;
    h.t.pad_id = s.pad_id;
    h.t.unk_id = s.unk_id;
    h.t.max_chars = s.max_input_chars;
    return nullptr;
}

inline size_t workspace_bytes(int max_chars, int B) { return static_cast<size_t>(B) * (max_chars + 1) * 8 + 256; }

// ================================================================ byte-level BPE (RoBERTa, ModernBERT, EuroBERT)
// Three kernels.  split: one thread per text matches the added tokens (normalized = false on the raw text, then
// normalized = true inside the gaps), runs the split pattern over each remaining gap and records up to max_length - 2 entries:
// an added token, or a word (a byte span, with ByteLevel's prefix space in front).  merge: one thread per word of the whole
// batch runs the library's BPE (lowest rank first, leftmost on ties) with a binary heap, O(n log n) in the word's bytes.
// gather: one warp per text lays the entries' tokens out as [CLS] tokens [SEP], truncated to max_length.  Every word yields
// at least one token (the vocab holds all 256 byte symbols), so max_length - 2 entries are all the kept words.
//
// A word longer than kMaxWord bytes is not merged on the device: its text is left to the caller (lengths = -1, and
// max_len[1] = 1), which tokenizes it on the host.  One GPU thread would otherwise run for a long time on one word.
constexpr int kMaxWord = AC_BPE_MAX_WORD;
enum { kSplitGpt2 = 0, kSplitLlama3 = 1 };
// bpe class bits of a codepoint (tokenizer.bpe_classes): \p{L}, \p{N}, \s of the library's regex engine, Rust whitespace
// (lstrip / rstrip); bits 4-7 the contraction letter it matches case-insensitively (1..8 = s t r e v m l d)
enum { kL = 1, kN = 2, kS = 4, kRust = 8 };
enum { kFoldS = 1, kFoldT, kFoldR, kFoldE, kFoldV, kFoldM, kFoldL, kFoldD };
// added-token trie node terminal codes: (added index << 2) | lstrip << 1 | rstrip, or -1
struct BpeTables {
    const uint8_t *cls;
    const int4 *merges;         // (left id, right id, rank, merged id); left < 0: empty
    uint32_t merge_mask;
    const int4 *words;          // ignore_merges: the model vocab over raw bytes, (id, hash, byte offset, byte length)
    uint32_t word_mask;
    const uint8_t *word_bytes;
    const int2 *edges;          // added-token trie edges: (node << 8 | byte, child); key < 0: empty
    uint32_t edge_mask;
    const int2 *term;           // per trie node: terminal code of the raw pass, of the normalized pass
    const int32_t *added_id;
    uint32_t first_byte[2][8];  // bit set: a token of the raw / normalized pass starts with this byte
    int n_pass[2];              // added tokens in each pass
    int byte_id[256];
    int split, prefix_space, ignore_merges;
    int cls_id, sep_id, pad_id;
};

// one gap's view of the text: bytes [a, b) relative to the text, with ByteLevel's prefix space as byte a - 1 when vp
struct Gap {
    const uint8_t *p;
    int64_t a, b;
    bool vp;
};

__device__ inline int gap_decode(const Gap &g, int64_t i, uint32_t &c) {
    if (i < g.a) { c = ' '; return 1; }
    return utf8_decode(g.p + i, g.p + g.b, c);
}

// a text's slots: slot 1 + j belongs to byte j, slot 0 to the prefix space of a word at byte 0; a word's tokens are written
// over its slots from its first one
struct Entries {
    int2 *e;                    // a word: (first slot, (bytes << 1) | vp); after the merge (first slot, -tokens).  (id, 0): an added token
    int n, limit;
    int64_t slots;              // slots the workspace holds for this text
    bool huge;                  // a kept word is longer than kMaxWord
};

__device__ inline void emit_word(Entries &o, const Gap &g, int64_t i, int64_t j) {
    if (o.n >= o.limit) return;
    if (j - i > kMaxWord) { o.huge = true; return; }
    const bool vp = i < g.a;
    const int64_t slot = i + 1;              // the prefix space is byte a - 1: its slot belongs to the token before the gap
    o.e[o.n++] = int2{static_cast<int>(slot), static_cast<int>(((j - i) << 1) | (vp ? 1 : 0))};
}

__device__ inline void emit_added(Entries &o, const BpeTables &t, int code) {
    if (o.n >= o.limit) return;
    o.e[o.n++] = int2{t.added_id[code >> 2], 0};
}

// the end of the run of codepoints from i whose class has any bit of `mask` (set: `want` true) or none (`want` false)
__device__ inline int64_t class_run(const BpeTables &t, const Gap &g, int64_t i, int mask, bool want, int64_t *last = nullptr) {
    while (i < g.b) {
        uint32_t c;
        const int n = gap_decode(g, i, c);
        if (((t.cls[c] & mask) != 0) != want) break;
        if (last) *last = i;
        i += n;
    }
    return i;
}

__device__ inline int64_t rn_run(const Gap &g, int64_t i) {
    while (i < g.b && (g.p[i] == '\r' || g.p[i] == '\n')) ++i;
    return i;
}

// the end of the match at i of the split pattern; every codepoint starts a match of either pattern
// G (GPT-2, ByteLevel use_regex): 's|'t|'re|'ve|'m|'ll|'d| ?\p{L}+| ?\p{N}+| ?[^\s\p{L}\p{N}]+|\s+(?!\S)|\s+
// L (Llama-3): (?i:'s|'t|'re|'ve|'m|'ll|'d)|[^\r\n\p{L}\p{N}]?\p{L}+|\p{N}{1,3}| ?[^\s\p{L}\p{N}]+[\r\n]*|\s*[\r\n]+|\s+(?!\S)|\s+
__device__ inline int64_t split_match(const BpeTables &t, const Gap &g, int64_t i) {
    const bool llama = t.split == kSplitLlama3;
    uint32_t c0, c1 = 0, c2 = 0;
    const int n0 = gap_decode(g, i, c0);
    const int64_t i1 = i + n0;
    const int n1 = i1 < g.b ? gap_decode(g, i1, c1) : 0;
    const int k0 = t.cls[c0], k1 = n1 ? t.cls[c1] : kS;     // past the end: no letter, number or other char follows
    if (c0 == '\'' && n1) {
        const int64_t i2 = i1 + n1;
        const int n2 = i2 < g.b ? gap_decode(g, i2, c2) : 0;
        if (llama) {
            const int f1 = k1 >> 4, f2 = n2 ? t.cls[c2] >> 4 : 0;
            if (f1 == kFoldS || f1 == kFoldT || f1 == kFoldM || f1 == kFoldD) return i2;
            if (((f1 == kFoldR || f1 == kFoldV) && f2 == kFoldE) || (f1 == kFoldL && f2 == kFoldL)) return i2 + n2;
        } else {
            if (c1 == 's' || c1 == 't' || c1 == 'm' || c1 == 'd') return i2;
            if (((c1 == 'r' || c1 == 'v') && c2 == 'e') || (c1 == 'l' && c2 == 'l')) return i2 + n2;
        }
    }
    const bool o0 = !(k0 & (kL | kN | kS)), o1 = n1 && !(k1 & (kL | kN | kS));
    if (llama) {
        if (!(k0 & (kL | kN)) && c0 != '\r' && c0 != '\n' && n1 && (k1 & kL)) return class_run(t, g, i1, kL, true);
        if (k0 & kL) return class_run(t, g, i, kL, true);
        if (k0 & kN) {
            int64_t j = i;
            for (int k = 0; k < 3 && j < g.b; ++k) {
                uint32_t c;
                const int n = gap_decode(g, j, c);
                if (!(t.cls[c] & kN)) break;
                j += n;
            }
            return j;
        }
        if (c0 == ' ' && o1) return rn_run(g, class_run(t, g, i1, kL | kN | kS, false));
        if (o0) return rn_run(g, class_run(t, g, i, kL | kN | kS, false));
    } else {
        if (c0 == ' ' && n1 && (k1 & kL)) return class_run(t, g, i1, kL, true);
        if (c0 == ' ' && n1 && (k1 & kN)) return class_run(t, g, i1, kN, true);
        if (c0 == ' ' && o1) return class_run(t, g, i1, kL | kN | kS, false);
        if (k0 & kL) return class_run(t, g, i, kL, true);
        if (k0 & kN) return class_run(t, g, i, kN, true);
        if (o0) return class_run(t, g, i, kL | kN | kS, false);
    }
    // c0 is whitespace: the run of it, which \s*[\r\n]+ (L) ends after its last \r or \n, and \s+(?!\S) before its last char
    // when a non-space follows
    int64_t last = i;
    const int64_t j = class_run(t, g, i, kS, true, &last);
    if (llama) {
        for (int64_t k = j - 1; k >= i && k >= g.a; --k)
            if (g.p[k] == '\r' || g.p[k] == '\n') return k + 1;
    }
    if (j == g.b || last == i) return j;
    return last;
}

// ByteLevel / Split over one gap: the words it yields, in order
__device__ inline void split_gap(const BpeTables &t, const uint8_t *p, int64_t a, int64_t b, Entries &o) {
    if (a >= b) return;                       // the library drops empty pieces before the pre-tokenizer runs
    Gap g{p, a, b, t.prefix_space && p[a] != ' '};
    for (int64_t i = g.vp ? a - 1 : a; i < b && o.n < o.limit && !o.huge;) {
        const int64_t j = split_match(t, g, i);
        emit_word(o, g, i, j);
        i = j;
    }
}

__device__ inline bool rust_space_at(const BpeTables &t, const uint8_t *p, int64_t i, int64_t end, int &n) {
    uint32_t c;
    n = utf8_decode(p + i, p + end, c);
    return (t.cls[c] & kRust) != 0;
}

// the child of `node` over `byte` in a byte trie whose edges (node << 8 | byte, child) sit in an open-addressing table, or -1
__host__ __device__ inline uint32_t trie_edge_hash(int key) {
    const uint32_t h = static_cast<uint32_t>(key) * 0x9E3779B1u;
    return h ^ (h >> 16);
}

__device__ inline int trie_child(const int2 *edges, uint32_t mask, int node, uint8_t byte) {
    const int key = (node << 8) | byte;
    for (uint32_t k = trie_edge_hash(key) & mask;; k = (k + 1) & mask) {
        const int2 x = edges[k];
        if (x.x < 0) return -1;
        if (x.x == key) return x.y;
    }
}

// the next added token of `pass` in [from, end) (aho-corasick leftmost-longest), widened by lstrip down to `from` and by
// rstrip up to `end` over Rust whitespace: returns its terminal code and [*s, *e), or -1 with *s = end
__device__ inline int next_added(const BpeTables &t, int pass, const uint8_t *p, int64_t from, int64_t end, int64_t *s,
                                 int64_t *e) {
    *s = end;
    if (!t.n_pass[pass]) return -1;
    for (int64_t i = from; i < end; ++i) {
        if (!((t.first_byte[pass][p[i] >> 5] >> (p[i] & 31)) & 1u)) continue;
        int node = 0, code = -1;
        int64_t stop = i;
        for (int64_t j = i; j < end; ++j) {
            node = trie_child(t.edges, t.edge_mask, node, p[j]);
            if (node < 0) break;
            const int2 tm = t.term[node];
            const int c = pass ? tm.y : tm.x;
            if (c >= 0) { code = c; stop = j + 1; }
        }
        if (code < 0) continue;
        int64_t a = i;
        int n;
        if (code & 2) {
            while (a > from) {
                int64_t q = a - 1;
                while (q > from && a - q < 4 && (p[q] & 0xC0) == 0x80) --q;
                if (!rust_space_at(t, p, q, a, n) || q + n != a) break;
                a = q;
            }
        }
        if (code & 1)
            while (stop < end && rust_space_at(t, p, stop, end, n)) stop += n;
        *s = a;
        *e = stop;
        return code;
    }
    return -1;
}

// entries of text b: ws_ent[b, 0 .. n_ent[b]); n_ent[b] = -1 and lengths[b] = -1 for a text left to the caller
__global__ void __launch_bounds__(128) tokenize_bpe_split_kernel(BpeTables t, const uint8_t *text, const int64_t *offsets,
                                                                 int B, int max_length, int64_t n_slots, int32_t *lengths,
                                                                 int32_t *max_len, int2 *ws_ent, int32_t *n_ent) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    const uint8_t *p = text + offsets[b];
    const int64_t len = offsets[b + 1] - offsets[b], base = offsets[b] - offsets[0] + b;
    const int limit = max_length - 2;
    Entries o{ws_ent + static_cast<int64_t>(b) * limit, 0, limit, n_slots - base, false};
    if (o.slots < len + 1 || len >= INT32_MAX) o.huge = true;       // the workspace was sized for fewer bytes
    for (int64_t g1 = 0; g1 <= len && o.n < o.limit && !o.huge;) {
        int64_t s1, e1;
        const int code1 = next_added(t, 0, p, g1, len, &s1, &e1);
        for (int64_t g2 = g1; o.n < o.limit && !o.huge;) {
            int64_t s2, e2;
            const int code2 = next_added(t, 1, p, g2, s1, &s2, &e2);
            split_gap(t, p, g2, s2, o);
            if (code2 < 0) break;
            emit_added(o, t, code2);
            g2 = e2;
        }
        if (code1 < 0 || o.huge) break;
        emit_added(o, t, code1);
        g1 = e1;
    }
    n_ent[b] = o.huge ? -1 : o.n;
    if (o.huge) {
        lengths[b] = -1;
        atomicMax(max_len + 1, 1);
    }
}

__device__ inline const int4 *merge_find(const BpeTables &t, int l, int r) {
    uint32_t h = static_cast<uint32_t>(l) * 0x9E3779B1u ^ static_cast<uint32_t>(r) * 0x85EBCA77u;
    h ^= h >> 15;
    for (uint32_t i = h & t.merge_mask;; i = (i + 1) & t.merge_mask) {
        const int4 *e = t.merges + i;
        if (e->x < 0) return nullptr;
        if (e->x == l && e->y == r) return e;
    }
}

__device__ inline int word_find(const BpeTables &t, const uint8_t *w, int n, bool vp) {
    uint32_t h = kFnvBasis;
    if (vp) h = (h ^ ' ') * 16777619u;
    h = fnv1a(h, w, n - vp);
    for (uint32_t i = h & t.word_mask;; i = (i + 1) & t.word_mask) {
        const int4 e = t.words[i];
        if (e.x < 0) return -1;
        if (static_cast<uint32_t>(e.y) != h || e.w != n) continue;
        const uint8_t *v = t.word_bytes + e.z;
        bool eq = !vp || v[0] == ' ';
        for (int j = 0; j < n - vp && eq; ++j) eq = v[vp + j] == w[j];
        if (eq) return e.x;
    }
}

__device__ inline void heap_push(uint64_t *h, int &n, uint64_t v) {
    int i = n++;
    while (i > 0) {
        const int up = (i - 1) >> 1;
        if (h[up] <= v) break;
        h[i] = h[up];
        i = up;
    }
    h[i] = v;
}

__device__ inline uint64_t heap_pop(uint64_t *h, int &n) {
    const uint64_t top = h[0], v = h[--n];
    int i = 0;
    for (;;) {
        int c = 2 * i + 1;
        if (c >= n) break;
        if (c + 1 < n && h[c + 1] < h[c]) ++c;
        if (v <= h[c]) break;
        h[i] = h[c];
        i = c;
    }
    if (n) h[i] = v;
    return top;
}

__device__ inline void push_pair(const BpeTables &t, uint64_t *h, int &hn, const int32_t *id, int pos, int right) {
    if (const int4 *m = merge_find(t, id[pos], id[right]))
        heap_push(h, hn, (static_cast<uint64_t>(static_cast<uint32_t>(m->z)) << 32) | static_cast<uint32_t>(pos));
}

// the BPE tokens of entry k of text b, written over the word's slots from its first one; its info becomes -(token count)
__global__ void __launch_bounds__(128) tokenize_bpe_merge_kernel(BpeTables t, const uint8_t *text, const int64_t *offsets,
                                                                 int B, int max_length, int2 *ws_ent, const int32_t *n_ent,
                                                                 int32_t *ws_tok, int32_t *ws_link, uint64_t *ws_heap) {
    const int limit = max_length - 2;
    const int64_t gid = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
    if (gid >= static_cast<int64_t>(B) * limit) return;
    const int b = static_cast<int>(gid / limit), k = static_cast<int>(gid - static_cast<int64_t>(b) * limit);
    if (k >= n_ent[b]) return;
    int2 &ent = ws_ent[gid];
    if (ent.y <= 0) return;
    const int n = ent.y >> 1;
    const bool vp = ent.y & 1;
    const int64_t base = offsets[b] - offsets[0] + b + ent.x;       // the word's first slot
    const uint8_t *w = text + offsets[b] + ent.x - 1 + vp;          // its first real byte
    int32_t *id = ws_tok + base;
    if (t.ignore_merges) {
        const int v = word_find(t, w, n, vp);
        if (v >= 0) {
            id[0] = v;
            ent.y = -1;
            return;
        }
    }
    for (int i = 0; i < n; ++i) id[i] = t.byte_id[(vp && i == 0) ? ' ' : w[i - vp]];
    if (n == 1) {
        ent.y = -1;
        return;
    }
    int32_t *next = ws_link + 2 * base, *prev = next + n;
    uint64_t *h = ws_heap + 3 * base;
    int hn = 0;
    for (int i = 0; i < n; ++i) {
        next[i] = i + 1 < n ? i + 1 : -1;
        prev[i] = i - 1;
    }
    for (int i = 0; i + 1 < n; ++i) push_pair(t, h, hn, id, i, i + 1);
    while (hn) {
        const uint64_t top = heap_pop(h, hn);
        const int pos = static_cast<int>(top & 0xffffffffu), rank = static_cast<int>(top >> 32);
        if (id[pos] < 0) continue;
        const int nx = next[pos];
        if (nx < 0) continue;
        const int4 *m = merge_find(t, id[pos], id[nx]);
        if (!m || m->z != rank) continue;                      // an entry for a pair that has changed since
        id[pos] = m->w;
        id[nx] = -1;
        const int nn = next[nx];
        next[pos] = nn;
        if (nn >= 0) prev[nn] = pos;
        if (prev[pos] >= 0) push_pair(t, h, hn, id, prev[pos], pos);
        if (nn >= 0) push_pair(t, h, hn, id, pos, nn);
    }
    int c = 0;
    for (int i = 0; i >= 0; i = next[i]) id[c++] = id[i];
    ent.y = -c;
}

// tokens[b] = [CLS] the entries' tokens [SEP], truncated to max_length; one warp per text.  Text b's slots start at
// (offsets[b] - offsets[0] + b) * slots_per_byte: one per byte and one more (BPE), or more (Unigram)
__global__ void __launch_bounds__(128) tokenize_bpe_gather_kernel(BpeTables t, const int64_t *offsets, int B, int max_length,
                                                                  const int2 *ws_ent, const int32_t *n_ent,
                                                                  const int32_t *ws_tok, int32_t *tokens, int32_t *lengths,
                                                                  int32_t *max_len, int slots_per_byte = 1) {
    const int b = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (b >= B) return;
    const int ne = n_ent[b];
    if (ne < 0) return;
    const int limit = max_length - 2;
    const int2 *ent = ws_ent + static_cast<int64_t>(b) * limit;
    const int32_t *slots = ws_tok + (offsets[b] - offsets[0] + b) * slots_per_byte;
    int32_t *row = tokens + static_cast<int64_t>(b) * max_length;
    int done = 0;
    for (int k0 = 0; k0 < ne && done < limit; k0 += 32) {
        const int k = k0 + lane;
        const int2 e = k < ne ? ent[k] : int2{0, 0};
        const int c = k < ne ? (e.y ? -e.y : 1) : 0;
        int incl = c;
        for (int d = 1; d < 32; d <<= 1) {
            const int v = __shfl_sync(0xffffffffu, incl, lane >= d ? lane - d : lane);
            if (lane >= d) incl += v;
        }
        for (int j = 0, at = done + incl - c; j < c && at + j < limit; ++j) row[1 + at + j] = e.y ? slots[e.x + j] : e.x;
        done += __shfl_sync(0xffffffffu, incl, 31);
    }
    if (lane == 0) {
        const int n = done < limit ? done : limit;
        row[0] = t.cls_id;
        row[1 + n] = t.sep_id;
        lengths[b] = n + 2;
        atomicMax(max_len, n + 2);
    }
}

// ---------------------------------------------------------------- host side of the BPE tables
struct BpeHost {
    std::vector<int4> merges, words;
    std::vector<int2> edges, term;
    std::vector<int32_t> added_id;
    BpeTables t{};              // scalars, byte ids and first_byte filled; pointers left to the owner
};

inline uint32_t pow2_at_least(size_t n) {
    size_t s = 2;
    while (s < n) s <<= 1;
    return static_cast<uint32_t>(s);
}

// a byte trie built on the host, nodes numbered from the root 0, laid out for trie_child
struct TrieBuilder {
    std::vector<std::vector<std::pair<int, int>>> kids{1};
    size_t n_edges = 0;
    int size() const { return static_cast<int>(kids.size()); }
    // the node of key s[0, n), created with its path; -1 once the trie outgrows the 2^23 nodes an edge key can name
    int insert(const uint8_t *s, int64_t n) {
        int node = 0;
        for (int64_t j = 0; j < n; ++j) {
            int child = -1;
            for (auto &e : kids[node])
                if (e.first == s[j]) child = e.second;
            if (child < 0) {
                child = static_cast<int>(kids.size());
                if (child >= (1 << 23)) return -1;
                kids[node].push_back({s[j], child});
                kids.emplace_back();
                ++n_edges;
            }
            node = child;
        }
        return node;
    }
    std::vector<int2> edges(uint32_t &mask) const {
        const uint32_t em = pow2_at_least(2 * n_edges);
        std::vector<int2> out(em, int2{-1, 0});
        for (size_t node = 0; node < kids.size(); ++node)
            for (auto &e : kids[node]) {
                const int key = static_cast<int>(node << 8) | e.first;
                uint32_t i = trie_edge_hash(key) & (em - 1);
                while (out[i].x >= 0) i = (i + 1) & (em - 1);
                out[i] = int2{key, e.second};
            }
        mask = em - 1;
        return out;
    }
};

// the added tokens into `trie`, with their terminal codes in h.term (one per node), first bytes and ids
inline const char *add_added_tokens(const uint8_t *bytes, const int64_t *offsets, const int32_t *ids, const uint8_t *flags,
                                    int n_added, TrieBuilder &trie, BpeHost &h) {
    h.term.assign(1, int2{-1, -1});
    memset(h.t.first_byte, 0, sizeof(h.t.first_byte));
    for (int a = 0; a < n_added; ++a) {
        const int64_t o0 = offsets[a], n = offsets[a + 1] - o0;
        if (n <= 0) return "empty added token";
        const int f = flags[a], pass = f & 1;
        const int node = trie.insert(bytes + o0, n);
        if (node < 0) return "added tokens too long";
        h.term.resize(trie.size(), int2{-1, -1});
        const int code = (a << 2) | (f & 2) | (f >> 2 & 1);     // lstrip << 1 | rstrip
        int &slot = pass ? h.term[node].y : h.term[node].x;
        if (slot < 0) slot = code;                    // the same content twice: the first one's id and flags
        h.t.first_byte[pass][bytes[o0] >> 5] |= 1u << (bytes[o0] & 31);
        ++h.t.n_pass[pass];
        h.added_id.push_back(ids[a]);
    }
    if (h.added_id.empty()) h.added_id.push_back(0);
    return nullptr;
}

inline const char *build_bpe_host_tables(const ac_bpe_tokenizer_spec &s, BpeHost &h) {
    if (!s.cls || !s.byte_ids || (s.n_merges && !s.merges) || s.n_merges < 0) return "null table";
    if (s.split != kSplitGpt2 && s.split != kSplitLlama3) return "unknown split pattern";
    if (s.ignore_merges && (!s.vocab_bytes || !s.vocab_offsets || !s.vocab_ids || s.n_vocab <= 0))
        return "ignore_merges without a vocab";
    if (s.n_added < 0 || (s.n_added && (!s.added_bytes || !s.added_offsets || !s.added_ids || !s.added_flags)))
        return "bad added tokens";
    for (int i = 0; i < 256; ++i) {
        if (s.byte_ids[i] < 0) return "a byte has no symbol in the vocab";
        h.t.byte_id[i] = s.byte_ids[i];
    }
    const uint32_t mm = pow2_at_least(2 * static_cast<size_t>(s.n_merges));
    h.merges.assign(mm, int4{-1, 0, 0, 0});
    for (int r = 0; r < s.n_merges; ++r) {
        const int l = s.merges[3 * r], rt = s.merges[3 * r + 1], nw = s.merges[3 * r + 2];
        if (l < 0 || rt < 0 || nw < 0) return "negative id in a merge";
        uint32_t x = static_cast<uint32_t>(l) * 0x9E3779B1u ^ static_cast<uint32_t>(rt) * 0x85EBCA77u;
        x ^= x >> 15;
        uint32_t i = x & (mm - 1);
        while (h.merges[i].x >= 0 && !(h.merges[i].x == l && h.merges[i].y == rt)) i = (i + 1) & (mm - 1);
        h.merges[i] = int4{l, rt, r, nw};            // a repeated pair keeps its last rank, as the library's map does
    }
    h.words.assign(2, int4{-1, 0, 0, 0});
    if (s.ignore_merges) {
        int max_key = 0;
        if (const char *why = hash_byte_strings(s.vocab_bytes, s.vocab_offsets, s.vocab_ids, s.n_vocab, h.words, max_key))
            return why;
    }
    TrieBuilder trie;
    if (const char *why = add_added_tokens(s.added_bytes, s.added_offsets, s.added_ids, s.added_flags, s.n_added, trie, h))
        return why;
    h.edges = trie.edges(h.t.edge_mask);
    h.t.merge_mask = mm - 1;
    h.t.word_mask = static_cast<uint32_t>(h.words.size() - 1);
    h.t.split = s.split;
    h.t.prefix_space = s.add_prefix_space ? 1 : 0;
    h.t.ignore_merges = s.ignore_merges ? 1 : 0;
    h.t.cls_id = s.cls_id;
    h.t.sep_id = s.sep_id;
    h.t.pad_id = s.pad_id;
    return nullptr;
}

// workspace of a BPE call, in this order: entries int2 [B, max_length - 2], n_ent int32 [B], then per slot (text bytes + B
// of them) the token / symbol id, the next and prev links and three heap entries
constexpr size_t kBpeSlotBytes = 4 + 8 + 24;
inline size_t bpe_fixed_bytes(int B, int max_length) {
    return (static_cast<size_t>(B) * (max_length - 2) * 8 + static_cast<size_t>(B) * 4 + 255) / 256 * 256;
}
inline size_t bpe_workspace_bytes(int B, int64_t text_bytes, int max_length) {
    return bpe_fixed_bytes(B, max_length) + (static_cast<size_t>(text_bytes) + B) * kBpeSlotBytes + 256;
}

// ================================================================ SentencePiece Unigram (XLM-RoBERTa, bge-m3, multilingual-e5)
// Two kernels of their own, then tokenize_bpe_gather_kernel.  split: one thread per text matches the added tokens as the BPE
// split does (normalized = false on the raw text; normalized = true on each gap after normalization), normalizes each gap
// with the Precompiled charsmap, splits it on whitespace and writes every word, "▁" in front unless it starts with one and
// cut before every later "▁" (Metaspace, prepend_scheme always, split), into the text's word area; at most max_length - 2
// entries.  viterbi: one thread per word of the whole batch runs the library's lattice over the word's char boundaries in
// fp64 and writes its tokens, consecutive unknown chars fused into one unk_id, over the word's slots.
//
// Precompiled, as the library runs it: the gap is cut into grapheme clusters; a cluster of fewer than 6 bytes that some key
// is a prefix of becomes the value of the shortest such key, whole; otherwise each char is replaced by its value when it is
// a key.  A word longer than kMaxUnigramWord bytes is not tokenized on the device: its text is left to the caller as in BPE.
constexpr int kMaxUnigramWord = AC_UNIGRAM_MAX_WORD;
constexpr int kPrecompiledCluster = 6;          // clusters this long or longer are normalized char by char
constexpr double kUnkPenalty = 10.0;            // an unknown char scores the lowest piece score minus this
constexpr uint32_t kMetaspace = 0x2581;
// unigram class bits of a codepoint (tokenizer.unigram_classes); kRust (8) is Rust whitespace as for BPE
enum { kJoin = 1, kControl = 2, kPrepend = 4 };

struct UnigramTables {
    BpeTables a;                // cls, the byte trie of the added tokens and the charsmap keys, added ids, special ids
    const int2 *map_val;        // per node of that trie: (offset, length) of the value of the key ending there; x < 0: none
    const uint8_t *map_pool;
    int n_map;                  // 0: no normalizer
    const int2 *piece_edges;    // byte trie of the pieces
    uint32_t piece_mask;
    const int32_t *piece_id;    // per piece-trie node: the id of the piece ending there, or -1
    const double *piece_score;
    int grow;                   // charsmap value bytes per key byte, at most (1 without a normalizer)
    int unk_id;
    double unk_score;
};

// per text: (bytes + 1) units; a unit holds `grow` bytes of one normalized gap and grow + 3 word slots (a slot: a word byte,
// its lattice node's score, start and id)
constexpr size_t kUniSlotBytes = 1 + 8 + 4 + 4;
inline size_t unigram_unit_bytes(int grow) { return (grow + 3) * kUniSlotBytes + grow; }
inline size_t unigram_workspace_bytes(int B, int64_t text_bytes, int max_length, int grow) {
    return bpe_fixed_bytes(B, max_length) + (static_cast<size_t>(text_bytes) + B) * unigram_unit_bytes(grow) + 256;
}

// a growing byte area of one text
struct Area {
    uint8_t *o;
    int64_t n, cap;
    bool over;
};

__device__ inline void area_put(Area &a, const uint8_t *s, int n) {
    if (a.n + n > a.cap) { a.over = true; return; }
    for (int i = 0; i < n; ++i) a.o[a.n + i] = s[i];
    a.n += n;
}

// the node of the shortest charsmap key that is a prefix of p[i, end), or -1
__device__ inline int map_prefix(const UnigramTables &t, const uint8_t *p, int64_t i, int64_t end) {
    int node = 0;
    for (int64_t j = i; j < end; ++j) {
        node = trie_child(t.a.edges, t.a.edge_mask, node, p[j]);
        if (node < 0) return -1;
        if (t.map_val[node].x >= 0) return node;
    }
    return -1;
}

// the end of the grapheme cluster at i, by the rules that can make one shorter than kPrecompiledCluster bytes: CR LF,
// nothing joins a control and a control joins nothing, Extend / ZWJ / SpacingMark join what precedes them, Prepend joins
// what follows it.  Emoji ZWJ sequences (GB11) are not modelled: "©" + ZWJ + "©" is cut after the ZWJ, where the library
// keeps one 7-byte cluster; the two differ only for a charsmap key that starts with © or ®, which unigram_spec refuses
__device__ inline int64_t cluster_end(const UnigramTables &t, const uint8_t *p, int64_t i, int64_t end) {
    uint32_t c;
    int64_t j = i + utf8_decode(p + i, p + end, c);
    if (c == '\r') return j < end && p[j] == '\n' ? j + 1 : j;
    int prev = t.a.cls[c];
    if (prev & kControl) return j;
    while (j < end) {
        uint32_t d;
        const int n = utf8_decode(p + j, p + end, d);
        const int k = t.a.cls[d];
        if ((k & kControl) || !((k & kJoin) || (prev & kPrepend))) break;
        j += n;
        prev = k;
    }
    return j;
}

__device__ inline void put_value(const UnigramTables &t, Area &o, int node) {
    const int2 v = t.map_val[node];
    area_put(o, t.map_pool + v.x, v.y);
}

// Precompiled over raw bytes [a, b) into o (valid UTF-8: an invalid byte becomes U+FFFD, as everywhere in this file)
__device__ inline void normalize_gap(const UnigramTables &t, const uint8_t *p, int64_t a, int64_t b, Area &o) {
    uint8_t buf[4];
    for (int64_t i = a; i < b && !o.over;) {
        const int64_t j = t.n_map ? cluster_end(t, p, i, b) : b;
        if (t.n_map && j - i < kPrecompiledCluster) {
            const int node = map_prefix(t, p, i, j);
            if (node >= 0) {
                put_value(t, o, node);
                i = j;
                continue;
            }
        }
        for (; i < j && !o.over;) {
            uint32_t c;
            const int n = utf8_decode(p + i, p + b, c);
            const int node = t.n_map ? map_prefix(t, p, i, i + n) : -1;
            if (node >= 0) put_value(t, o, node);
            else area_put(o, buf, utf8_encode(c, buf));
            i += n;
        }
    }
}

// WhitespaceSplit + Metaspace over normalized bytes [a, b) of g: each word into the word area w, one entry each
__device__ inline void split_words(const UnigramTables &t, const uint8_t *g, int64_t a, int64_t b, Area &w,
                                   Entries &o) {
    const uint8_t meta[3] = {0xE2, 0x96, 0x81};
    int64_t start = -1;
    for (int64_t i = a; i <= b && !o.huge;) {
        uint32_t c = ' ';
        const int n = i < b ? utf8_decode(g + i, g + b, c) : 1;
        const bool space = i == b || (t.a.cls[c] & kRust);
        if (start >= 0 && (space || c == kMetaspace)) {               // the word ends
            const int64_t len = w.n - start;
            if (len > kMaxUnigramWord) { o.huge = true; return; }
            o.e[o.n++] = int2{static_cast<int>(start), static_cast<int>(len)};
            start = -1;
        }
        if (!space) {
            if (start < 0) {
                if (o.n >= o.limit) return;
                start = w.n;
                if (c != kMetaspace) area_put(w, meta, 3);
            }
            area_put(w, g + i, n);
            if (w.over) { o.huge = true; return; }
        }
        i += n;
    }
}

// entries of text b: ws_ent[b, 0 .. n_ent[b]), words as (first slot, bytes) in the text's word area; n_ent[b] = -1 and
// lengths[b] = -1 for a text left to the caller
__global__ void __launch_bounds__(128) tokenize_unigram_split_kernel(UnigramTables t, const uint8_t *text,
                                                                     const int64_t *offsets, int B, int max_length,
                                                                     int64_t n_units, int32_t *lengths, int32_t *max_len,
                                                                     int2 *ws_ent, int32_t *n_ent, uint8_t *ws_words,
                                                                     uint8_t *ws_gap) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    const uint8_t *p = text + offsets[b];
    const int64_t len = offsets[b + 1] - offsets[b], unit = offsets[b] - offsets[0] + b;
    const int limit = max_length - 2;
    Entries o{ws_ent + static_cast<int64_t>(b) * limit, 0, limit, 0, false};
    Area w{ws_words + unit * (t.grow + 3), 0, (len + 1) * (t.grow + 3), false};
    Area g{ws_gap + unit * t.grow, 0, (len + 1) * t.grow, false};
    if (unit + len + 1 > n_units || len >= INT32_MAX / (t.grow + 3)) o.huge = true;   // the workspace holds fewer units
    for (int64_t g1 = 0; g1 <= len && o.n < o.limit && !o.huge;) {
        int64_t s1, e1;
        const int code1 = next_added(t.a, 0, p, g1, len, &s1, &e1);
        g.n = 0;
        normalize_gap(t, p, g1, s1, g);
        if (g.over) o.huge = true;
        for (int64_t g2 = 0; o.n < o.limit && !o.huge;) {
            int64_t s2, e2;
            const int code2 = next_added(t.a, 1, g.o, g2, g.n, &s2, &e2);
            split_words(t, g.o, g2, s2, w, o);
            if (code2 < 0) break;
            emit_added(o, t.a, code2);
            g2 = e2;
        }
        if (code1 < 0 || o.huge) break;
        emit_added(o, t.a, code1);
        g1 = e1;
    }
    n_ent[b] = o.huge ? -1 : o.n;
    if (o.huge) {
        lengths[b] = -1;
        atomicMax(max_len + 1, 1);
    }
}

// the Unigram tokens of entry k of text b (tokenizers' Unigram::encode_optimized): char boundaries left to right, pieces
// from each shortest first, a candidate kept only when strictly better; a char no one-char piece covers is unk.  The node
// of the best path ending after byte e sits at slot e; the tokens are written back to front over the word's last slots,
// which never reach a node still to be read.  The entry becomes (its first token's slot, -tokens).
__global__ void __launch_bounds__(128) tokenize_unigram_viterbi_kernel(UnigramTables t, const int64_t *offsets, int B,
                                                                       int max_length, int2 *ws_ent, const int32_t *n_ent,
                                                                       const uint8_t *ws_words, double *ws_score,
                                                                       int32_t *ws_start, int32_t *ws_tok) {
    const int limit = max_length - 2;
    const int64_t gid = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
    if (gid >= static_cast<int64_t>(B) * limit) return;
    const int b = static_cast<int>(gid / limit), k = static_cast<int>(gid - static_cast<int64_t>(b) * limit);
    if (k >= n_ent[b]) return;
    int2 &ent = ws_ent[gid];
    if (ent.y <= 0) return;
    const int n = ent.y;
    const int64_t base = (offsets[b] - offsets[0] + b) * (t.grow + 3) + ent.x;
    const uint8_t *w = ws_words + base;
    double *sc = ws_score + base;
    int32_t *st = ws_start + base, *id = ws_tok + base;
    for (int e = 0; e < n; ++e) st[e] = -1;
    for (int s = 0; s < n;) {
        const double here = s ? sc[s - 1] : 0.0;
        const uint8_t lead = w[s];
        const int mblen = std::min(lead < 0x80 ? 1 : lead >= 0xF0 ? 4 : lead >= 0xE0 ? 3 : 2, n - s);
        bool single = false;
        int node = 0;
        for (int e = s; e < n; ++e) {
            node = trie_child(t.piece_edges, t.piece_mask, node, w[e]);
            if (node < 0) break;
            const int v = t.piece_id[node];
            if (v < 0) continue;
            const double cand = here + t.piece_score[node];
            if (st[e] < 0 || cand > sc[e]) { sc[e] = cand; st[e] = s; id[e] = v; }
            if (e + 1 - s == mblen) single = true;
        }
        if (!single) {
            const int e = s + mblen - 1;
            const double cand = here + t.unk_score;
            if (st[e] < 0 || cand > sc[e]) { sc[e] = cand; st[e] = s; id[e] = t.unk_id; }
        }
        s += mblen;
    }
    int c = 0;
    bool unk = false;
    for (int e = n; e > 0;) {
        const int s = st[e - 1], v = id[e - 1];
        if (!(unk && v == t.unk_id)) id[n - 1 - c++] = v;
        unk = v == t.unk_id;
        e = s;
    }
    ent.x += n - c;
    ent.y = -c;
}

// ---------------------------------------------------------------- host side of the Unigram tables
struct UnigramHost {
    BpeHost a;                  // the added tokens' terminal codes, edges (charsmap keys too) and ids
    std::vector<int2> map_val, piece_edges;
    std::vector<uint8_t> map_pool;
    std::vector<int32_t> piece_id;
    std::vector<double> piece_score;
    UnigramTables t{};          // scalars filled; pointers left to the owner
};

inline const char *build_unigram_host_tables(const ac_unigram_tokenizer_spec &s, UnigramHost &h) {
    if (!s.cls || !s.piece_bytes || !s.piece_offsets || !s.piece_scores || s.n_pieces <= 0) return "null table or no pieces";
    if (s.n_map < 0 || (s.n_map && (!s.map_keys || !s.map_key_offsets || !s.map_values || !s.map_value_offsets)))
        return "bad charsmap";
    if (s.grow < 1 || s.grow > 64) return "charsmap expansion outside 1..64 bytes per byte";
    if (s.unk_id < 0 || s.unk_id >= s.n_pieces) return "unk_id outside the pieces";
    if (s.n_added < 0 || (s.n_added && (!s.added_bytes || !s.added_offsets || !s.added_ids || !s.added_flags)))
        return "bad added tokens";
    TrieBuilder trie;
    if (const char *why = add_added_tokens(s.added_bytes, s.added_offsets, s.added_ids, s.added_flags, s.n_added, trie, h.a))
        return why;
    for (int k = 0; k < s.n_map; ++k) {
        const int64_t k0 = s.map_key_offsets[k], kn = s.map_key_offsets[k + 1] - k0;
        const int64_t v0 = s.map_value_offsets[k], vn = s.map_value_offsets[k + 1] - v0;
        if (kn <= 0 || vn < 0 || vn > s.grow * kn) return "empty charsmap key, or a value longer than grow allows";
        const int node = trie.insert(s.map_keys + k0, kn);
        if (node < 0) return "charsmap too large";
        h.map_val.resize(trie.size(), int2{-1, 0});
        if (h.map_pool.size() + vn > INT32_MAX) return "charsmap values over 2 GB";
        h.map_val[node] = int2{static_cast<int>(h.map_pool.size()), static_cast<int>(vn)};
        h.map_pool.insert(h.map_pool.end(), s.map_values + v0, s.map_values + v0 + vn);
    }
    h.map_val.resize(trie.size(), int2{-1, 0});
    h.a.term.resize(trie.size(), int2{-1, -1});
    if (h.map_pool.empty()) h.map_pool.push_back(0);
    h.a.edges = trie.edges(h.a.t.edge_mask);
    // the pieces: the library keeps the last id of a repeated piece, and its score; the lowest score of all sets unk's
    TrieBuilder pieces;
    double lowest = 0.0;
    for (int v = 0; v < s.n_pieces; ++v) {
        const int64_t o0 = s.piece_offsets[v], n = s.piece_offsets[v + 1] - o0;
        if (n <= 0) return "empty piece";
        const int node = pieces.insert(s.piece_bytes + o0, n);
        if (node < 0) return "pieces too large";
        h.piece_id.resize(pieces.size(), -1);
        h.piece_score.resize(pieces.size(), 0.0);
        h.piece_id[node] = v;
        h.piece_score[node] = s.piece_scores[v];
        lowest = v ? std::min(lowest, s.piece_scores[v]) : s.piece_scores[v];
    }
    h.piece_id.resize(pieces.size(), -1);
    h.piece_score.resize(pieces.size(), 0.0);
    h.piece_edges = pieces.edges(h.t.piece_mask);
    h.t.a = h.a.t;
    h.t.a.cls_id = s.cls_id;
    h.t.a.sep_id = s.sep_id;
    h.t.a.pad_id = s.pad_id;
    h.t.n_map = s.n_map;
    h.t.grow = s.grow;
    h.t.unk_id = s.unk_id;
    h.t.unk_score = lowest - kUnkPenalty;
    return nullptr;
}

}  // namespace tok
}  // namespace ac

#ifndef AC_CPU_SHIM
using namespace ac;

// one handle type for every kind: `kind` tells which table set the calls read
enum TokKind { kWordPiece, kBpe, kUnigram };
struct ac_tokenizer {
    TokKind kind;
    tok::Tables t;
    tok::BpeTables b;
    tok::UnigramTables u;
    int pad_id;
    std::vector<void *> owned;
};

static int tok_upload(ac_tokenizer *k, const void *src, size_t bytes, const void **dst) {
    void *d = nullptr;
    AC_CUDA(cudaMalloc(&d, bytes ? bytes : 1));
    k->owned.push_back(d);
    if (bytes) AC_CUDA(cudaMemcpy(d, src, bytes, cudaMemcpyHostToDevice));
    *dst = d;
    return AC_OK;
}

extern "C" int ac_tokenizer_destroy(ac_tokenizer *tok) {
    if (!tok) return AC_OK;
    for (void *p : tok->owned) cudaFree(p);
    delete tok;
    return AC_OK;
}

extern "C" int ac_tokenizer_create(const ac_tokenizer_spec *spec, ac_tokenizer **out) {
    AC_REQUIRE(spec && out, "ac_tokenizer_create: null argument");
    *out = nullptr;
    tok::HostTables h;
    if (const char *why = tok::build_host_tables(*spec, h)) {
        set_error("ac_tokenizer_create: %s", why);
        return AC_E_INVALID;
    }
    ac_tokenizer *k = new ac_tokenizer();
    k->kind = kWordPiece;
    k->t = h.t;
    k->pad_id = h.t.pad_id;
    const void *p[8];
    int rc = AC_OK;
    const int64_t vbytes = spec->vocab_offsets[spec->n_vocab];
    if ((rc = tok_upload(k, spec->norm, sizeof(uint32_t) * tok::kCodepoints, &p[0])) ||
        (rc = tok_upload(k, spec->cls, tok::kCodepoints, &p[1])) ||
        (rc = tok_upload(k, spec->pool, sizeof(uint32_t) * spec->pool_len, &p[2])) ||
        (rc = tok_upload(k, h.slots.data(), sizeof(int4) * h.slots.size(), &p[3])) ||
        (rc = tok_upload(k, spec->vocab_bytes, vbytes, &p[4])) ||
        (rc = tok_upload(k, h.added_bytes.data(), h.added_bytes.size(), &p[5])) ||
        (rc = tok_upload(k, h.added_off.data(), sizeof(int64_t) * h.added_off.size(), &p[6])) ||
        (rc = tok_upload(k, h.added_id.data(), sizeof(int32_t) * h.added_id.size(), &p[7]))) {
        ac_tokenizer_destroy(k);
        return rc;
    }
    k->t.norm = static_cast<const uint32_t *>(p[0]);
    k->t.cls = static_cast<const uint8_t *>(p[1]);
    k->t.pool = static_cast<const uint32_t *>(p[2]);
    k->t.slots = static_cast<const int4 *>(p[3]);
    k->t.vocab_bytes = static_cast<const uint8_t *>(p[4]);
    k->t.added_bytes = static_cast<const uint8_t *>(p[5]);
    k->t.added_off = static_cast<const int64_t *>(p[6]);
    k->t.added_id = static_cast<const int32_t *>(p[7]);
    *out = k;
    return AC_OK;
}

extern "C" int ac_tokenizer_create_bpe(const ac_bpe_tokenizer_spec *spec, ac_tokenizer **out) {
    AC_REQUIRE(spec && out, "ac_tokenizer_create_bpe: null argument");
    *out = nullptr;
    tok::BpeHost h;
    if (const char *why = tok::build_bpe_host_tables(*spec, h)) {
        set_error("ac_tokenizer_create_bpe: %s", why);
        return AC_E_INVALID;
    }
    ac_tokenizer *k = new ac_tokenizer();
    k->kind = kBpe;
    k->b = h.t;
    k->pad_id = h.t.pad_id;
    const void *p[7];
    int rc = AC_OK;
    const int64_t vbytes = spec->ignore_merges ? spec->vocab_offsets[spec->n_vocab] : 0;
    if ((rc = tok_upload(k, spec->cls, tok::kCodepoints, &p[0])) ||
        (rc = tok_upload(k, h.merges.data(), sizeof(int4) * h.merges.size(), &p[1])) ||
        (rc = tok_upload(k, h.words.data(), sizeof(int4) * h.words.size(), &p[2])) ||
        (rc = tok_upload(k, spec->vocab_bytes, vbytes, &p[3])) ||
        (rc = tok_upload(k, h.edges.data(), sizeof(int2) * h.edges.size(), &p[4])) ||
        (rc = tok_upload(k, h.term.data(), sizeof(int2) * h.term.size(), &p[5])) ||
        (rc = tok_upload(k, h.added_id.data(), sizeof(int32_t) * h.added_id.size(), &p[6]))) {
        ac_tokenizer_destroy(k);
        return rc;
    }
    k->b.cls = static_cast<const uint8_t *>(p[0]);
    k->b.merges = static_cast<const int4 *>(p[1]);
    k->b.words = static_cast<const int4 *>(p[2]);
    k->b.word_bytes = static_cast<const uint8_t *>(p[3]);
    k->b.edges = static_cast<const int2 *>(p[4]);
    k->b.term = static_cast<const int2 *>(p[5]);
    k->b.added_id = static_cast<const int32_t *>(p[6]);
    *out = k;
    return AC_OK;
}

extern "C" int ac_tokenizer_create_unigram(const ac_unigram_tokenizer_spec *spec, ac_tokenizer **out) {
    AC_REQUIRE(spec && out, "ac_tokenizer_create_unigram: null argument");
    *out = nullptr;
    tok::UnigramHost h;
    if (const char *why = tok::build_unigram_host_tables(*spec, h)) {
        set_error("ac_tokenizer_create_unigram: %s", why);
        return AC_E_INVALID;
    }
    ac_tokenizer *k = new ac_tokenizer();
    k->kind = kUnigram;
    k->u = h.t;
    k->pad_id = spec->pad_id;
    const void *p[10];
    int rc = AC_OK;
    if ((rc = tok_upload(k, spec->cls, tok::kCodepoints, &p[0])) ||
        (rc = tok_upload(k, h.a.edges.data(), sizeof(int2) * h.a.edges.size(), &p[1])) ||
        (rc = tok_upload(k, h.a.term.data(), sizeof(int2) * h.a.term.size(), &p[2])) ||
        (rc = tok_upload(k, h.a.added_id.data(), sizeof(int32_t) * h.a.added_id.size(), &p[3])) ||
        (rc = tok_upload(k, h.map_val.data(), sizeof(int2) * h.map_val.size(), &p[4])) ||
        (rc = tok_upload(k, h.map_pool.data(), h.map_pool.size(), &p[5])) ||
        (rc = tok_upload(k, h.piece_edges.data(), sizeof(int2) * h.piece_edges.size(), &p[6])) ||
        (rc = tok_upload(k, h.piece_id.data(), sizeof(int32_t) * h.piece_id.size(), &p[7])) ||
        (rc = tok_upload(k, h.piece_score.data(), sizeof(double) * h.piece_score.size(), &p[8]))) {
        ac_tokenizer_destroy(k);
        return rc;
    }
    k->u.a.cls = static_cast<const uint8_t *>(p[0]);
    k->u.a.edges = static_cast<const int2 *>(p[1]);
    k->u.a.term = static_cast<const int2 *>(p[2]);
    k->u.a.added_id = static_cast<const int32_t *>(p[3]);
    k->u.map_val = static_cast<const int2 *>(p[4]);
    k->u.map_pool = static_cast<const uint8_t *>(p[5]);
    k->u.piece_edges = static_cast<const int2 *>(p[6]);
    k->u.piece_id = static_cast<const int32_t *>(p[7]);
    k->u.piece_score = static_cast<const double *>(p[8]);
    *out = k;
    return AC_OK;
}

extern "C" int ac_tokenize_workspace_bytes(const ac_tokenizer *tok, int B, size_t *bytes) {
    AC_REQUIRE(tok && bytes && B >= 0, "ac_tokenize_workspace_bytes: bad arguments");
    AC_REQUIRE(tok->kind == kWordPiece, "ac_tokenize_workspace_bytes: a %s handle's workspace depends on the text bytes; use "
               "ac_tokenize_workspace_bytes_text", tok->kind == kBpe ? "BPE" : "Unigram");
    *bytes = tok::workspace_bytes(tok->t.max_chars, B);
    return AC_OK;
}

extern "C" int ac_tokenize_workspace_bytes_text(const ac_tokenizer *tok, int B, int64_t text_bytes, int max_length,
                                                size_t *bytes) {
    AC_REQUIRE(tok && bytes && B >= 0 && text_bytes >= 0 && max_length >= 2, "ac_tokenize_workspace_bytes_text: bad arguments");
    *bytes = tok->kind == kBpe       ? tok::bpe_workspace_bytes(B, text_bytes, max_length)
             : tok->kind == kUnigram ? tok::unigram_workspace_bytes(B, text_bytes, max_length, tok->u.grow)
                                     : tok::workspace_bytes(tok->t.max_chars, B);
    return AC_OK;
}

static int tokenize_bpe(const ac_tokenizer *tok, const uint8_t *text, const int64_t *offsets, int B, int max_length,
                        int32_t *tokens, int32_t *lengths, int32_t *max_len, void *workspace, size_t workspace_bytes,
                        cudaStream_t s) {
    const size_t fixed = tok::bpe_fixed_bytes(B, max_length);
    AC_REQUIRE(workspace && workspace_bytes >= tok::bpe_workspace_bytes(B, 0, max_length), "ac_tokenize: workspace too small");
    // the slots the workspace holds; a text past them is left to the caller like a text with a huge word
    const int64_t n_slots = static_cast<int64_t>((workspace_bytes - fixed - 256) / tok::kBpeSlotBytes);
    int2 *ent = static_cast<int2 *>(workspace);
    int32_t *n_ent = reinterpret_cast<int32_t *>(ent + static_cast<size_t>(B) * (max_length - 2));
    int32_t *ws_tok = reinterpret_cast<int32_t *>(static_cast<uint8_t *>(workspace) + fixed);
    int32_t *ws_link = ws_tok + n_slots;
    uint64_t *ws_heap = reinterpret_cast<uint64_t *>(reinterpret_cast<uintptr_t>(ws_link + 2 * n_slots + 1) & ~uintptr_t(7));
    AC_CUDA(cudaMemsetAsync(max_len, 0, 2 * sizeof(int32_t), s));
    tok::tokenize_bpe_split_kernel<<<(B + 127) / 128, 128, 0, s>>>(tok->b, text, offsets, B, max_length, n_slots, lengths,
                                                                   max_len, ent, n_ent);
    AC_LAUNCH_CHECK();
    const int64_t words = static_cast<int64_t>(B) * (max_length - 2);
    if (words) {
        tok::tokenize_bpe_merge_kernel<<<static_cast<unsigned>((words + 127) / 128), 128, 0, s>>>(
            tok->b, text, offsets, B, max_length, ent, n_ent, ws_tok, ws_link, ws_heap);
        AC_LAUNCH_CHECK();
    }
    tok::tokenize_bpe_gather_kernel<<<(B + 3) / 4, 128, 0, s>>>(tok->b, offsets, B, max_length, ent, n_ent, ws_tok, tokens,
                                                                lengths, max_len);
    AC_LAUNCH_CHECK();
    return AC_OK;
}

static int tokenize_unigram(const ac_tokenizer *tok, const uint8_t *text, const int64_t *offsets, int B, int max_length,
                            int32_t *tokens, int32_t *lengths, int32_t *max_len, void *workspace, size_t workspace_bytes,
                            cudaStream_t s) {
    const tok::UnigramTables &u = tok->u;
    const size_t fixed = tok::bpe_fixed_bytes(B, max_length);
    AC_REQUIRE(workspace && workspace_bytes >= tok::unigram_workspace_bytes(B, 0, max_length, u.grow),
               "ac_tokenize: workspace too small");
    // the units the workspace holds; a text past them is left to the caller like a text with a huge word
    const int64_t n_units = static_cast<int64_t>((workspace_bytes - fixed - 256) / tok::unigram_unit_bytes(u.grow));
    const int64_t n_slots = n_units * (u.grow + 3);
    int2 *ent = static_cast<int2 *>(workspace);
    int32_t *n_ent = reinterpret_cast<int32_t *>(ent + static_cast<size_t>(B) * (max_length - 2));
    double *ws_score = reinterpret_cast<double *>(static_cast<uint8_t *>(workspace) + fixed);
    int32_t *ws_start = reinterpret_cast<int32_t *>(ws_score + n_slots);
    int32_t *ws_tok = ws_start + n_slots;
    uint8_t *ws_words = reinterpret_cast<uint8_t *>(ws_tok + n_slots);
    uint8_t *ws_gap = ws_words + n_slots;
    AC_CUDA(cudaMemsetAsync(max_len, 0, 2 * sizeof(int32_t), s));
    tok::tokenize_unigram_split_kernel<<<(B + 127) / 128, 128, 0, s>>>(u, text, offsets, B, max_length, n_units, lengths,
                                                                       max_len, ent, n_ent, ws_words, ws_gap);
    AC_LAUNCH_CHECK();
    const int64_t words = static_cast<int64_t>(B) * (max_length - 2);
    if (words) {
        tok::tokenize_unigram_viterbi_kernel<<<static_cast<unsigned>((words + 127) / 128), 128, 0, s>>>(
            u, offsets, B, max_length, ent, n_ent, ws_words, ws_score, ws_start, ws_tok);
        AC_LAUNCH_CHECK();
    }
    tok::tokenize_bpe_gather_kernel<<<(B + 3) / 4, 128, 0, s>>>(u.a, offsets, B, max_length, ent, n_ent, ws_tok, tokens,
                                                                lengths, max_len, u.grow + 3);
    AC_LAUNCH_CHECK();
    return AC_OK;
}

extern "C" int ac_tokenize(const ac_tokenizer *tok, const uint8_t *text, const int64_t *offsets, int B, int max_length,
                           int32_t *tokens, int32_t *lengths, int32_t *max_len, void *workspace, size_t workspace_bytes,
                           ac_stream_t stream) {
    AC_REQUIRE(tok && text && offsets && tokens && lengths && max_len && B >= 1, "ac_tokenize: bad arguments");
    AC_REQUIRE(max_length >= 2, "ac_tokenize: max_length=%d < 2 leaves no room for the two special tokens", max_length);
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (tok->kind == kUnigram)
        return tokenize_unigram(tok, text, offsets, B, max_length, tokens, lengths, max_len, workspace, workspace_bytes, s);
    if (tok->kind == kBpe) return tokenize_bpe(tok, text, offsets, B, max_length, tokens, lengths, max_len, workspace, workspace_bytes, s);
    AC_REQUIRE(workspace && workspace_bytes >= tok::workspace_bytes(tok->t.max_chars, B), "ac_tokenize: workspace too small");
    uint32_t *ws_cp = static_cast<uint32_t *>(workspace);
    uint8_t *ws_bytes = reinterpret_cast<uint8_t *>(ws_cp + static_cast<size_t>(B) * (tok->t.max_chars + 1));
    AC_CUDA(cudaMemsetAsync(max_len, 0, sizeof(int32_t), s));
    tok::tokenize_wordpiece_kernel<<<(B + 127) / 128, 128, 0, s>>>(tok->t, text, offsets, B, max_length, tokens, lengths,
                                                                   max_len, ws_cp, ws_bytes);
    AC_LAUNCH_CHECK();
    return AC_OK;
}

extern "C" int ac_tokenize_pack(const ac_tokenizer *tok, const int32_t *tokens, const int32_t *lengths, int B, int max_length,
                                int S, int32_t *ids, int32_t *mask, int32_t *type_ids, ac_stream_t stream) {
    AC_REQUIRE(tok && tokens && lengths && ids && mask && B >= 1 && S >= 1 && S <= max_length, "ac_tokenize_pack: bad arguments");
    const int64_t total = static_cast<int64_t>(B) * S;
    const int grid = static_cast<int>(std::min<int64_t>((total + 255) / 256, 4 * sm_count()));
    tok::tokenize_pack_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(tokens, lengths, B, max_length, S,
                                                                                   tok->pad_id, ids, mask, type_ids);
    AC_LAUNCH_CHECK();
    return AC_OK;
}
#endif
