// Host build of the SentencePiece-style BPE stages of smg_b200/csrc: the ▁ normalization, the segmenter and the character-level symbolizer
// (metaspace.cuh) and the merge loop (bpe.cuh merge_symbols), compiled with g++ so that tests/test_metaspace_host.py can compare exactly the
// code the kernels run with live `tokenizers`.
//   test_metaspace_host <prepend: 0 never, 1 first, 2 always, 3 legacy> <split: 0 | 1>
// stdin, all integers u32 little-endian: the model — n_tokens, then (id, byte length, bytes) per token; n_merges, then (left id, right id)
// pairs in priority order; n_specials, then (id, byte length, bytes) — followed by records of (byte length, UTF-8 bytes).
// stdout, two lines per record: "P <ids>" from the pieces the GPU merges independently (cut at the stretch start and before every ▁ that
// follows another character, or before every ▁ with split), "W <ids>" with every stretch merged as one word (what `tokenizers` does).
// The vocabulary tables are laid out as Tokenizer::build lays them out (open addressing, same hashes).
#include <cstdint>
#include <cstdio>
#include <string>
#include <unordered_map>
#include <vector>

#include "metaspace.cuh"

using namespace smgx;

static uint32_t rd() {
    uint32_t x = 0;
    if (std::fread(&x, 4, 1, stdin) != 1) { std::fprintf(stderr, "short input\n"); std::exit(2); }
    return x;
}
static std::string rd_str() {
    std::string s(rd(), '\0');
    if (!s.empty() && std::fread(&s[0], 1, s.size(), stdin) != s.size()) std::exit(2);
    return s;
}
static uint32_t pow2_at_least(uint64_t x) { uint32_t p = 1024; while (p < x) p <<= 1; return p; }

struct HostModel {
    std::vector<uint32_t> byte_token = std::vector<uint32_t>(256, 0);
    std::vector<PairSlot> pairs;
    std::vector<PieceSlot> pieces;
    std::vector<uint8_t> blob;
    std::vector<SpecialTok> specials;
    BpeView v{};
};

static void load(HostModel& M) {
    std::unordered_map<std::string, uint32_t> enc;
    std::unordered_map<uint32_t, std::string> by_id;
    uint32_t max_len = 1;
    for (uint32_t n = rd(), k = 0; k < n; ++k) {
        const uint32_t id = rd();
        const std::string s = rd_str();
        enc[s] = id;
        by_id[id] = s;
        max_len = std::max<uint32_t>(max_len, (uint32_t)s.size());
    }
    for (int b = 0; b < 256; ++b) {
        char name[8];
        std::snprintf(name, sizeof(name), "<0x%02X>", b);
        M.byte_token[b] = enc.at(name);
    }
    M.pieces.assign(pow2_at_least(enc.size() * 2), PieceSlot{0, 0, 0, 0, 0});
    const uint32_t pmask = (uint32_t)M.pieces.size() - 1;
    for (auto& kv : enc) {
        const uint32_t off = (uint32_t)M.blob.size();
        M.blob.insert(M.blob.end(), kv.first.begin(), kv.first.end());
        const uint64_t hsh = bytes_hash((const uint8_t*)kv.first.data(), (uint32_t)kv.first.size());
        uint32_t h = (uint32_t)(hsh >> 32) & pmask;
        while (M.pieces[h].hash) h = (h + 1) & pmask;
        M.pieces[h] = PieceSlot{hsh, kv.second, (uint32_t)kv.first.size(), off, 0};
    }
    const uint32_t n_merges = rd();
    M.pairs.assign(pow2_at_least((uint64_t)n_merges * 2 + 2), PairSlot{kPairEmpty, kRankMax, 0});
    const uint32_t qmask = (uint32_t)M.pairs.size() - 1;
    for (uint32_t k = 0; k < n_merges; ++k) {
        const uint32_t l = rd(), r = rd();
        const uint64_t key = ((uint64_t)l << 32) | r;
        const uint32_t id = enc.at(by_id.at(l) + by_id.at(r));
        uint32_t h = (uint32_t)(mix64(key) >> 32) & qmask;
        while (M.pairs[h].key != kPairEmpty && M.pairs[h].key != key) h = (h + 1) & qmask;
        if (M.pairs[h].key == key) continue;   // a repeated pair keeps its first priority
        M.pairs[h] = PairSlot{key, k, id};
    }
    uint32_t first_bits[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (uint32_t n = rd(), k = 0; k < n; ++k) {
        const uint32_t id = rd();
        const std::string s = rd_str();
        M.specials.push_back(SpecialTok{(uint32_t)M.blob.size(), (uint32_t)s.size(), id, 0});
        M.blob.insert(M.blob.end(), s.begin(), s.end());
        first_bits[(uint8_t)s[0] >> 5] |= 1u << ((uint8_t)s[0] & 31);
    }
    BpeView& v = M.v;
    v.byte_token = M.byte_token.data();
    v.pairs = M.pairs.data();
    v.pair_mask = qmask;
    v.pieces = M.pieces.data();
    v.piece_mask = pmask;
    v.blob = M.blob.data();
    v.max_token_len = max_len;
    v.specials = M.specials.data();
    v.n_special = (uint32_t)M.specials.size();
    for (int i = 0; i < 8; ++i) v.special_first[i] = first_bits[i];
}

static void print(const char* tag, const std::vector<uint32_t>& ids) {
    std::fputs(tag, stdout);
    for (uint32_t x : ids) std::printf(" %u", x);
    std::fputc('\n', stdout);
}

// merge the symbols of slots [a, b) of tmp (kMsInvalid between them) and append the tokens
static void merge_span(const BpeView& v, const std::vector<uint32_t>& tmp, uint32_t a, uint32_t b, std::vector<uint32_t>& out) {
    std::vector<uint32_t> sym;
    for (uint32_t j = a; j < b; ++j) if (tmp[j] != kMsInvalid) sym.push_back(tmp[j]);
    std::vector<uint64_t> rk(sym.size() + 1);
    const uint32_t m = merge_symbols(v, sym.data(), (uint32_t)sym.size(), rk.data());
    out.insert(out.end(), sym.begin(), sym.begin() + m);
}

static void encode(const HostModel& M, const MetaspaceMode& mm, const std::string& text) {
    const BpeView& v = M.v;
    const uint8_t* s = (const uint8_t*)text.data();
    const uint32_t n = (uint32_t)text.size();
    // specials on the raw text, leftmost then longest (special_candidates_kernel + special_resolve_kernel)
    std::vector<uint8_t> flags(n + 1, 0);
    std::vector<uint32_t> sid(n + 1, kMsInvalid);
    for (uint32_t i = 0; i < n;) {
        uint32_t len, id;
        if (special_at(v, s, i, n, len, id)) {
            for (uint32_t j = 0; j < len; ++j) flags[i + j] = j ? 3 : 2;
            sid[i] = id;
            i += len;
        } else ++i;
    }
    // normalization (ms_count_kernel / ms_write_kernel)
    std::vector<uint8_t> nt(6 * (size_t)n + 8, 0), nf(6 * (size_t)n + 8, 0);
    std::vector<uint32_t> tmp(6 * (size_t)n + 8, kMsInvalid);
    uint32_t o = 0;
    for (uint32_t i = 0; i < n; ++i) {
        const uint32_t len = ms_out_write(mm, s, flags.data(), i, 0, &nt[o]);
        if (len != ms_out_len(mm, s, flags.data(), i, 0)) { std::fprintf(stderr, "ms_out_len disagrees with ms_out_write\n"); std::exit(3); }
        for (uint32_t j = 0; j < len; ++j) nf[o + j] = flags[i] >= 2 ? flags[i] : 0;
        if (flags[i] >= 2) tmp[o] = sid[i];
        o += len;
    }
    const uint32_t nn = o;
    // symbolizer + segmenter (ms_symbolize_kernel)
    for (uint32_t i = 0; i < nn; ++i) {
        if (nf[i] >= 2 || (nt[i] & 0xC0) == 0x80) continue;
        uint32_t ns;
        ms_symbolize(v, nt.data(), i, nn, &tmp[i], &ns);
        if (ms_piece_start(nt.data(), nf.data(), i, 0, mm.split)) nf[i] = 1;
    }
    // P: every piece merged on its own (ms_emit_kernel + the merge tiers); W: every stretch as one word
    std::vector<uint32_t> P, W;
    for (uint32_t i = 0; i < nn;) {
        if (nf[i] >= 2) {
            if (nf[i] == 2) { P.push_back(tmp[i]); W.push_back(tmp[i]); }
            ++i;
            continue;
        }
        uint32_t e = i + 1;
        while (e < nn && nf[e] < 2) ++e;   // the stretch [i, e)
        merge_span(v, tmp, i, e, W);
        for (uint32_t a = i; a < e;) {
            uint32_t b = a + 1;
            while (b < e && nf[b] != 1) ++b;
            merge_span(v, tmp, a, b, P);
            a = b;
        }
        i = e;
    }
    print("P", P);
    print("W", W);
}

int main(int argc, char** argv) {
    if (argc < 3) { std::fprintf(stderr, "usage: %s <prepend 0-3> <split 0|1>\n", argv[0]); return 2; }
    const MetaspaceMode mm{1, (uint32_t)std::atoi(argv[1]), (uint32_t)std::atoi(argv[2])};
    HostModel M;
    load(M);
    uint32_t len;
    while (std::fread(&len, 4, 1, stdin) == 1) {
        std::string text(len, '\0');
        if (len && std::fread(&text[0], 1, len, stdin) != len) return 2;
        encode(M, mm, text);
    }
    return 0;
}
