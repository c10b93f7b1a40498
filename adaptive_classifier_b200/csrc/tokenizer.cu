// tokenizer.cu -- WordPiece tokenization on the device for BERT-family tokenizers (BertNormalizer + BertPreTokenizer +
// WordPiece + "[special] A [special]"), ids identical to the Hugging Face `tokenizers` pipeline (adaptive_classifier_b200/
// tokenizer.py decides which tokenizers qualify and builds the Unicode tables by probing the installed library).
//
// One thread per text walks its UTF-8 bytes once: added tokens (normalized = false) are matched on the raw bytes, every other
// codepoint is replaced by its normalized expansion (table), the expansion's codepoints are split into words by their
// pre-tokenizer class (table), and each finished word is cut by greedy longest-match WordPiece against an open-addressing hash
// table of the vocab.  The walk stops once max_length - 2 tokens exist: later words cannot change the kept ids.
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

// returns nullptr, or what is wrong with the spec
inline const char *build_host_tables(const ac_tokenizer_spec &s, HostTables &h) {
    if (!s.norm || !s.cls || (s.pool_len && !s.pool) || !s.vocab_bytes || !s.vocab_offsets || !s.vocab_ids || s.n_vocab <= 0)
        return "null table or empty vocab";
    if (s.prefix_len < 0 || s.prefix_len > kMaxPrefix || (s.prefix_len && !s.prefix)) return "continuing_subword_prefix longer than 16 bytes";
    if (s.max_input_chars < 1) return "max_input_chars_per_word < 1";
    if (s.n_added < 0 || (s.n_added && (!s.added_bytes || !s.added_offsets || !s.added_ids))) return "bad added tokens";
    if (s.pool_len > (kOffsetMask >> 5)) return "expansion pool too large";
    size_t n_slots = 2;
    while (n_slots < 2 * static_cast<size_t>(s.n_vocab)) n_slots <<= 1;      // load factor <= 1/2: every probe chain ends
    h.slots.assign(n_slots, int4{-1, 0, 0, 0});
    int max_key = 0;
    for (int v = 0; v < s.n_vocab; ++v) {
        const int64_t o0 = s.vocab_offsets[v], n = s.vocab_offsets[v + 1] - o0;
        if (n <= 0 || o0 + n > INT32_MAX) return "empty vocab entry or vocab bytes over 2 GB";
        const uint32_t hash = fnv1a(kFnvBasis, s.vocab_bytes + o0, static_cast<int>(n));
        size_t i = hash & (n_slots - 1);
        while (h.slots[i].x >= 0) {
            const int4 &e = h.slots[i];
            if (e.w == n && !memcmp(s.vocab_bytes + e.z, s.vocab_bytes + o0, n)) return "duplicate vocab entry";
            i = (i + 1) & (n_slots - 1);
        }
        if (s.vocab_ids[v] < 0) return "negative vocab id";
        h.slots[i] = int4{s.vocab_ids[v], static_cast<int>(hash), static_cast<int>(o0), static_cast<int>(n)};
        max_key = std::max<int>(max_key, static_cast<int>(n));
    }
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

}  // namespace tok
}  // namespace ac

#ifndef AC_CPU_SHIM
using namespace ac;

struct ac_tokenizer {
    tok::Tables t;
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
    k->t = h.t;
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

extern "C" int ac_tokenize_workspace_bytes(const ac_tokenizer *tok, int B, size_t *bytes) {
    AC_REQUIRE(tok && bytes && B >= 0, "ac_tokenize_workspace_bytes: bad arguments");
    *bytes = tok::workspace_bytes(tok->t.max_chars, B);
    return AC_OK;
}

extern "C" int ac_tokenize(const ac_tokenizer *tok, const uint8_t *text, const int64_t *offsets, int B, int max_length,
                           int32_t *tokens, int32_t *lengths, int32_t *max_len, void *workspace, size_t workspace_bytes,
                           ac_stream_t stream) {
    AC_REQUIRE(tok && text && offsets && tokens && lengths && max_len && B >= 1, "ac_tokenize: bad arguments");
    AC_REQUIRE(max_length >= 2, "ac_tokenize: max_length=%d < 2 leaves no room for the two special tokens", max_length);
    AC_REQUIRE(workspace && workspace_bytes >= tok::workspace_bytes(tok->t.max_chars, B), "ac_tokenize: workspace too small");
    cudaStream_t s = static_cast<cudaStream_t>(stream);
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
                                                                                   tok->t.pad_id, ids, mask, type_ids);
    AC_LAUNCH_CHECK();
    return AC_OK;
}
#endif
