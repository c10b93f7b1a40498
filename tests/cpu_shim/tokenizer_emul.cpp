// tokenizer_emul.cpp -- TEST INFRASTRUCTURE.  Runs the kernels of csrc/tokenizer.cu ON THE CPU through tests/cpu_shim/cuda_shim.h
// (every CUDA thread a fiber, thread order shuffled by the seed), with the tables built by the same host code as
// ac_tokenizer_create.
//   usage: tokenizer_emul in.bin out.bin seed
//   in.bin: int64 records, each a length n then n bytes (padded to 8): norm, cls, pool, vocab bytes, vocab offsets, vocab ids,
//           added bytes, added offsets, added ids, prefix, then int64 scalars cls sep pad unk max_chars B max_length, then the
//           text bytes and the text offsets.  out.bin: int32 tokens [B, max_length], lengths [B], max_len, then the packed
//           ids / mask / type_ids [B, max_len].
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
    v.resize(n + 8);
    return v;
}

int main(int argc, char **argv) {
    if (argc != 4) { fprintf(stderr, "usage: tokenizer_emul in.bin out.bin seed\n"); return 2; }
    FILE *f = fopen(argv[1], "rb");
    std::vector<uint8_t> rec[10];
    for (auto &r : rec) r = record(f);
    int64_t sc[7];
    if (fread(sc, 8, 7, f) != 7) return 2;
    std::vector<uint8_t> text = record(f), off_b = record(f);
    fclose(f);
    const int B = static_cast<int>(sc[5]), max_length = static_cast<int>(sc[6]);
    const int64_t *voff = reinterpret_cast<const int64_t *>(rec[4].data());
    ac_tokenizer_spec s{};
    s.norm = reinterpret_cast<const uint32_t *>(rec[0].data());
    s.cls = rec[1].data();
    s.pool = reinterpret_cast<const uint32_t *>(rec[2].data());
    s.pool_len = static_cast<int64_t>(rec[2].size() - 8) / 4;
    s.vocab_bytes = rec[3].data();
    s.vocab_offsets = voff;
    s.vocab_ids = reinterpret_cast<const int32_t *>(rec[5].data());
    s.n_vocab = static_cast<int>((rec[5].size() - 8) / 4);
    s.added_bytes = rec[6].data();
    s.added_offsets = reinterpret_cast<const int64_t *>(rec[7].data());
    s.added_ids = reinterpret_cast<const int32_t *>(rec[8].data());
    s.n_added = static_cast<int>((rec[8].size() - 8) / 4);
    s.prefix = reinterpret_cast<const char *>(rec[9].data());
    s.prefix_len = static_cast<int>(rec[9].size() - 8);
    s.cls_id = static_cast<int>(sc[0]); s.sep_id = static_cast<int>(sc[1]); s.pad_id = static_cast<int>(sc[2]);
    s.unk_id = static_cast<int>(sc[3]); s.max_input_chars = static_cast<int>(sc[4]);
    HostTables h;
    if (const char *why = build_host_tables(s, h)) { fprintf(stderr, "tables: %s\n", why); return 3; }
    Tables t = h.t;
    t.norm = s.norm; t.cls = s.cls; t.pool = s.pool; t.slots = h.slots.data(); t.vocab_bytes = s.vocab_bytes;
    t.added_bytes = h.added_bytes.data(); t.added_off = h.added_off.data(); t.added_id = h.added_id.data();
    const int64_t *toff = reinterpret_cast<const int64_t *>(off_b.data());
    std::vector<uint8_t> text_exact(text.begin(), text.begin() + toff[B]);   // no slack after the last text (sanitizer builds)
    std::vector<int32_t> tokens(static_cast<size_t>(B) * max_length, -7), lengths(B, -7);
    int32_t max_len = 0;
    std::vector<uint8_t> ws(workspace_bytes(t.max_chars, B));
    uint32_t *ws_cp = reinterpret_cast<uint32_t *>(ws.data());
    uint8_t *ws_bytes = reinterpret_cast<uint8_t *>(ws_cp + static_cast<size_t>(B) * (t.max_chars + 1));
    const unsigned seed = static_cast<unsigned>(atoi(argv[3]));
    shim::launch(dim3((B + 127) / 128), dim3(128), [&] {
        tokenize_wordpiece_kernel(t, text_exact.data(), toff, B, max_length, tokens.data(), lengths.data(), &max_len, ws_cp, ws_bytes);
    }, seed);
    const int S = max_len;
    std::vector<int32_t> ids(static_cast<size_t>(B) * S), mask(ids.size()), tt(ids.size(), -7);
    shim::launch(dim3(3), dim3(64), [&] {
        tokenize_pack_kernel(tokens.data(), lengths.data(), B, max_length, S, t.pad_id, ids.data(), mask.data(), tt.data());
    }, seed + 1);
    FILE *o = fopen(argv[2], "wb");
    fwrite(tokens.data(), 4, tokens.size(), o);
    fwrite(lengths.data(), 4, lengths.size(), o);
    fwrite(&max_len, 4, 1, o);
    fwrite(ids.data(), 4, ids.size(), o);
    fwrite(mask.data(), 4, mask.size(), o);
    fwrite(tt.data(), 4, tt.size(), o);
    fclose(o);
    return 0;
}
