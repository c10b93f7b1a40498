// tokenizer_unigram_emul.cpp -- TEST INFRASTRUCTURE.  Runs the SentencePiece Unigram kernels of csrc/tokenizer.cu ON THE CPU
// through tests/cpu_shim/cuda_shim.h (every CUDA thread a fiber, thread order shuffled by the seed), with the tables built by
// the same host code as ac_tokenizer_create_unigram and a workspace of exactly ac_tokenize_workspace_bytes_text bytes.
//   usage: tokenizer_unigram_emul in.bin out.bin seed
//   in.bin: int64 records, each a length n then n bytes (padded to 8): cls, charsmap keys, key offsets, values, value
//           offsets, piece bytes, piece offsets, piece scores, added bytes, added offsets, added ids, added flags, then int64
//           scalars grow unk cls sep pad B max_length mode, then the text bytes and the text offsets.
//   out.bin, mode 0: int32 tokens [B, max_length], lengths [B], max_len [2], then the packed ids / mask [B, max_len[0]].
//   out.bin, mode 1 (Precompiled alone, each text one gap): per text an int64 length (-1: over the workspace) and the bytes.
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
    if (argc != 4) { fprintf(stderr, "usage: tokenizer_unigram_emul in.bin out.bin seed\n"); return 2; }
    FILE *f = fopen(argv[1], "rb");
    std::vector<uint8_t> rec[12];
    for (auto &r : rec) r = record(f);
    int64_t sc[8];
    if (fread(sc, 8, 8, f) != 8) return 2;
    std::vector<uint8_t> text = record(f), off_b = record(f);
    fclose(f);
    const int B = static_cast<int>(sc[5]), max_length = static_cast<int>(sc[6]), mode = static_cast<int>(sc[7]);
    ac_unigram_tokenizer_spec s{};
    s.cls = rec[0].data();
    s.map_keys = rec[1].data();
    s.map_key_offsets = reinterpret_cast<const int64_t *>(rec[2].data());
    s.map_values = rec[3].data();
    s.map_value_offsets = reinterpret_cast<const int64_t *>(rec[4].data());
    s.n_map = static_cast<int>(rec[2].size() / 8) - 1;
    s.piece_bytes = rec[5].data();
    s.piece_offsets = reinterpret_cast<const int64_t *>(rec[6].data());
    s.piece_scores = reinterpret_cast<const double *>(rec[7].data());
    s.n_pieces = static_cast<int>(rec[7].size() / 8);
    s.added_bytes = rec[8].data();
    s.added_offsets = reinterpret_cast<const int64_t *>(rec[9].data());
    s.added_ids = reinterpret_cast<const int32_t *>(rec[10].data());
    s.added_flags = rec[11].data();
    s.n_added = static_cast<int>(rec[10].size() / 4);
    s.grow = static_cast<int>(sc[0]);
    s.unk_id = static_cast<int>(sc[1]);
    s.cls_id = static_cast<int>(sc[2]); s.sep_id = static_cast<int>(sc[3]); s.pad_id = static_cast<int>(sc[4]);
    UnigramHost h;
    if (const char *why = build_unigram_host_tables(s, h)) { fprintf(stderr, "tables: %s\n", why); return 3; }
    UnigramTables t = h.t;
    t.a.cls = s.cls; t.a.edges = h.a.edges.data(); t.a.term = h.a.term.data(); t.a.added_id = h.a.added_id.data();
    t.map_val = h.map_val.data(); t.map_pool = h.map_pool.data();
    t.piece_edges = h.piece_edges.data(); t.piece_id = h.piece_id.data(); t.piece_score = h.piece_score.data();
    const int64_t *toff = reinterpret_cast<const int64_t *>(off_b.data());
    std::vector<uint8_t> text_exact(text.begin(), text.begin() + toff[B]);   // no slack after the last text (sanitizer builds)
    const int64_t text_bytes = toff[B] - toff[0];
    const unsigned seed = static_cast<unsigned>(atoi(argv[3]));
    FILE *o = fopen(argv[2], "wb");
    if (mode == 1) {
        std::vector<std::vector<uint8_t>> outs(B);
        std::vector<int64_t> lens(B);
        for (int b = 0; b < B; ++b) outs[b].resize(static_cast<size_t>(toff[b + 1] - toff[b] + 1) * t.grow);
        shim::launch(dim3((B + 127) / 128), dim3(128), [&] {
            const int b = blockIdx.x * blockDim.x + threadIdx.x;
            if (b >= B) return;
            Area a{outs[b].data(), 0, static_cast<int64_t>(outs[b].size()), false};
            normalize_gap(t, text_exact.data() + toff[b], 0, toff[b + 1] - toff[b], a);
            lens[b] = a.over ? -1 : a.n;
        }, seed);
        for (int b = 0; b < B; ++b) {
            fwrite(&lens[b], 8, 1, o);
            if (lens[b] > 0) fwrite(outs[b].data(), 1, lens[b], o);
        }
        fclose(o);
        return 0;
    }
    const size_t wsb = unigram_workspace_bytes(B, text_bytes, max_length, t.grow), fixed = bpe_fixed_bytes(B, max_length);
    std::vector<uint64_t> ws_store((wsb + 7) / 8);
    uint8_t *ws = reinterpret_cast<uint8_t *>(ws_store.data());
    const int64_t n_units = static_cast<int64_t>((wsb - fixed - 256) / unigram_unit_bytes(t.grow));
    const int64_t n_slots = n_units * (t.grow + 3);
    int2 *ent = reinterpret_cast<int2 *>(ws);
    int32_t *n_ent = reinterpret_cast<int32_t *>(ent + static_cast<size_t>(B) * (max_length - 2));
    double *ws_score = reinterpret_cast<double *>(ws + fixed);
    int32_t *ws_start = reinterpret_cast<int32_t *>(ws_score + n_slots);
    int32_t *ws_tok = ws_start + n_slots;
    uint8_t *ws_words = reinterpret_cast<uint8_t *>(ws_tok + n_slots);
    uint8_t *ws_gap = ws_words + n_slots;
    std::vector<int32_t> tokens(static_cast<size_t>(B) * max_length, -7), lengths(B, -7);
    int32_t max_len[2] = {0, 0};
    shim::launch(dim3((B + 127) / 128), dim3(128), [&] {
        tokenize_unigram_split_kernel(t, text_exact.data(), toff, B, max_length, n_units, lengths.data(), max_len, ent, n_ent,
                                      ws_words, ws_gap);
    }, seed);
    const int64_t words = static_cast<int64_t>(B) * (max_length - 2);
    if (words)
        shim::launch(dim3(static_cast<unsigned>((words + 127) / 128)), dim3(128), [&] {
            tokenize_unigram_viterbi_kernel(t, toff, B, max_length, ent, n_ent, ws_words, ws_score, ws_start, ws_tok);
        }, seed + 1);
    shim::launch(dim3((B + 3) / 4), dim3(128), [&] {
        tokenize_bpe_gather_kernel(t.a, toff, B, max_length, ent, n_ent, ws_tok, tokens.data(), lengths.data(), max_len,
                                   t.grow + 3);
    }, seed + 2);
    const int S = max_len[0];
    std::vector<int32_t> ids(static_cast<size_t>(B) * S), mask(ids.size());
    if (S)
        shim::launch(dim3(3), dim3(64), [&] {
            tokenize_pack_kernel(tokens.data(), lengths.data(), B, max_length, S, t.a.pad_id, ids.data(), mask.data(), nullptr);
        }, seed + 3);
    fwrite(tokens.data(), 4, tokens.size(), o);
    fwrite(lengths.data(), 4, lengths.size(), o);
    fwrite(max_len, 4, 2, o);
    fwrite(ids.data(), 4, ids.size(), o);
    fwrite(mask.data(), 4, mask.size(), o);
    fclose(o);
    return 0;
}
