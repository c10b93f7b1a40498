// tokenizer_bpe_emul.cpp -- TEST INFRASTRUCTURE.  Runs the byte-level BPE kernels of csrc/tokenizer.cu ON THE CPU through
// tests/cpu_shim/cuda_shim.h (every CUDA thread a fiber, thread order shuffled by the seed), with the tables built by the same
// host code as ac_tokenizer_create_bpe and a workspace of exactly ac_tokenize_workspace_bytes_text bytes.
//   usage: tokenizer_bpe_emul in.bin out.bin seed
//   in.bin: int64 records, each a length n then n bytes (padded to 8): cls, vocab bytes, vocab offsets, vocab ids, byte ids,
//           merges, added bytes, added offsets, added ids, added flags, then int64 scalars split add_prefix_space
//           ignore_merges cls sep pad B max_length mode, then the text bytes and the text offsets.
//   out.bin, mode 0: int32 tokens [B, max_length], lengths [B], max_len [2], then the packed ids / mask / type_ids [B, max_len[0]].
//   out.bin, mode 1 (the split stage alone): int32 n_ent [B], then the entries int2 [B, max_length - 2].
#include "cuda_shim.h"
#define AC_CPU_SHIM 1
#include "../../include/adaptive_b200.h"
static inline int atomicMax(int *p, int v) {          // fibers switch only inside barriers: a plain read-modify-write is atomic
    const int o = *p;
    if (v > o) *p = v;
    return o;
}
#include "../../adaptive_classifier_b200/csrc/tokenizer.cu"

using namespace ac::tok;

static std::vector<uint8_t> record(FILE *f) {
    int64_t n = 0;
    if (fread(&n, 8, 1, f) != 1) { fprintf(stderr, "truncated input\n"); exit(2); }
    std::vector<uint8_t> v(static_cast<size_t>((n + 7) / 8 * 8) + 8);
    if (n && fread(v.data(), 1, (n + 7) / 8 * 8, f) != static_cast<size_t>((n + 7) / 8 * 8)) { fprintf(stderr, "truncated\n"); exit(2); }
    v.resize(n);
    return v;
}

int main(int argc, char **argv) {
    if (argc != 4) { fprintf(stderr, "usage: tokenizer_bpe_emul in.bin out.bin seed\n"); return 2; }
    FILE *f = fopen(argv[1], "rb");
    std::vector<uint8_t> rec[10];
    for (auto &r : rec) r = record(f);
    int64_t sc[9];
    if (fread(sc, 8, 9, f) != 9) return 2;
    std::vector<uint8_t> text = record(f), off_b = record(f);
    fclose(f);
    const int B = static_cast<int>(sc[6]), max_length = static_cast<int>(sc[7]), mode = static_cast<int>(sc[8]);
    ac_bpe_tokenizer_spec s{};
    s.cls = rec[0].data();
    s.split = static_cast<int>(sc[0]);
    s.add_prefix_space = static_cast<int>(sc[1]);
    s.ignore_merges = static_cast<int>(sc[2]);
    s.vocab_bytes = rec[1].data();
    s.vocab_offsets = reinterpret_cast<const int64_t *>(rec[2].data());
    s.vocab_ids = reinterpret_cast<const int32_t *>(rec[3].data());
    s.n_vocab = static_cast<int>(rec[3].size() / 4);
    s.byte_ids = reinterpret_cast<const int32_t *>(rec[4].data());
    s.merges = reinterpret_cast<const int32_t *>(rec[5].data());
    s.n_merges = static_cast<int>(rec[5].size() / 12);
    s.added_bytes = rec[6].data();
    s.added_offsets = reinterpret_cast<const int64_t *>(rec[7].data());
    s.added_ids = reinterpret_cast<const int32_t *>(rec[8].data());
    s.added_flags = rec[9].data();
    s.n_added = static_cast<int>(rec[8].size() / 4);
    s.cls_id = static_cast<int>(sc[3]); s.sep_id = static_cast<int>(sc[4]); s.pad_id = static_cast<int>(sc[5]);
    BpeHost h;
    if (const char *why = build_bpe_host_tables(s, h)) { fprintf(stderr, "tables: %s\n", why); return 3; }
    BpeTables t = h.t;
    t.cls = s.cls; t.merges = h.merges.data(); t.words = h.words.data(); t.word_bytes = s.vocab_bytes;
    t.edges = h.edges.data(); t.term = h.term.data(); t.added_id = h.added_id.data();
    const int64_t *toff = reinterpret_cast<const int64_t *>(off_b.data());
    std::vector<uint8_t> text_exact(text.begin(), text.begin() + toff[B]);   // no slack after the last text (sanitizer builds)
    const int64_t text_bytes = toff[B] - toff[0];
    const size_t wsb = bpe_workspace_bytes(B, text_bytes, max_length), fixed = bpe_fixed_bytes(B, max_length);
    std::vector<uint64_t> ws_store((wsb + 7) / 8);
    uint8_t *ws = reinterpret_cast<uint8_t *>(ws_store.data());
    const int64_t n_slots = static_cast<int64_t>((wsb - fixed - 256) / kBpeSlotBytes);
    int2 *ent = reinterpret_cast<int2 *>(ws);
    int32_t *n_ent = reinterpret_cast<int32_t *>(ent + static_cast<size_t>(B) * (max_length - 2));
    int32_t *ws_tok = reinterpret_cast<int32_t *>(ws + fixed);
    int32_t *ws_link = ws_tok + n_slots;
    uint64_t *ws_heap = reinterpret_cast<uint64_t *>(reinterpret_cast<uintptr_t>(ws_link + 2 * n_slots + 1) & ~uintptr_t(7));
    std::vector<int32_t> tokens(static_cast<size_t>(B) * max_length, -7), lengths(B, -7);
    int32_t max_len[2] = {0, 0};
    const unsigned seed = static_cast<unsigned>(atoi(argv[3]));
    shim::launch(dim3((B + 127) / 128), dim3(128), [&] {
        tokenize_bpe_split_kernel(t, text_exact.data(), toff, B, max_length, n_slots, lengths.data(), max_len, ent, n_ent);
    }, seed);
    FILE *o = fopen(argv[2], "wb");
    if (mode == 1) {
        fwrite(n_ent, 4, B, o);
        fwrite(ent, 8, static_cast<size_t>(B) * (max_length - 2), o);
        fclose(o);
        return 0;
    }
    const int64_t words = static_cast<int64_t>(B) * (max_length - 2);
    if (words)
        shim::launch(dim3(static_cast<unsigned>((words + 127) / 128)), dim3(128), [&] {
            tokenize_bpe_merge_kernel(t, text_exact.data(), toff, B, max_length, ent, n_ent, ws_tok, ws_link, ws_heap);
        }, seed + 1);
    shim::launch(dim3((B + 3) / 4), dim3(128), [&] {
        tokenize_bpe_gather_kernel(t, toff, B, max_length, ent, n_ent, ws_tok, tokens.data(), lengths.data(), max_len);
    }, seed + 2);
    const int S = max_len[0];
    std::vector<int32_t> ids(static_cast<size_t>(B) * S), mask(ids.size()), tt(ids.size(), -7);
    if (S)
        shim::launch(dim3(3), dim3(64), [&] {
            tokenize_pack_kernel(tokens.data(), lengths.data(), B, max_length, S, t.pad_id, ids.data(), mask.data(), tt.data());
        }, seed + 3);
    fwrite(tokens.data(), 4, tokens.size(), o);
    fwrite(lengths.data(), 4, lengths.size(), o);
    fwrite(max_len, 4, 2, o);
    fwrite(ids.data(), 4, ids.size(), o);
    fwrite(mask.data(), 4, mask.size(), o);
    fwrite(tt.data(), 4, tt.size(), o);
    fclose(o);
    return 0;
}
