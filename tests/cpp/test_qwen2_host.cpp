// Host build of the Qwen2 tokenizer.json pieces of smg_b200/csrc: the Qwen2 pre-tokenizer (bpe.cuh) and the NFC normalizer (nfc.cuh),
// compiled with g++ so that tests/test_qwen2_host.py can compare exactly the code the kernels run with `regex` and `tokenizers`.
// stdin: records of (u32 little-endian byte length, UTF-8 bytes).
//   test_qwen2_host split  → three lines per record: "S <piece starts of the serial split>", "A <anchors>", "G <starts of the anchored
//                            split the GPU kernel does: from every anchor, replay the matcher up to the next anchor>"
//   test_qwen2_host nfc    → two records per record, same framing: the NFC the GPU stage computes (cut at NFC-stable code points, each
//                            segment in a 32-entry buffer or, when longer, with the counting sort), then the whole text as one segment
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "nfc.cuh"
#include "nfc_tables.h"
#include "unicode_tables.h"

using namespace smgx;

static const NfcView kNfc{kNfcCccCp, kNfcCccVal, kNfcCccN, kNfcDecCp, kNfcDecOff, kNfcDecData, kNfcDecN,
                          kNfcCompKey, kNfcCompVal, kNfcCompN, kNfcUnstLo, kNfcUnstHi, kNfcUnstableN};

static void print(const char* tag, const std::vector<uint32_t>& v) {
    std::fputs(tag, stdout);
    for (uint32_t x : v) std::printf(" %u", x);
    std::fputc('\n', stdout);
}

static void split(const uint8_t* s, uint32_t len) {
    const UnicodeView u{kUniLo, kUniHi, kUniCls, kUniRanges};
    std::vector<uint32_t> starts, anchors, seg;
    for (uint32_t i = 0; i < len; i = next_piece_qwen2(s, i, len, u)) starts.push_back(i);
    std::vector<uint8_t> is_anchor(len, 0);
    for (uint32_t i = 0; i < len; ++i)
        if ((s[i] & 0xC0) != 0x80 && is_anchor_qwen2(s, i, 0, nullptr, u)) { anchors.push_back(i); is_anchor[i] = 1; }
    for (uint32_t p : anchors)
        do { seg.push_back(p); p = next_piece_qwen2(s, p, len, u); } while (p < len && !is_anchor[p]);
    print("S", starts);
    print("A", anchors);
    print("G", seg);
}

static std::string whole(const uint8_t* s, uint32_t n) {
    static uint32_t hist[256];
    std::vector<uint32_t> e(4 * (size_t)n + 4);
    const uint32_t cap = 2 * n + 2;
    uint32_t m = nfc_decompose_text(kNfc, s, 0, n, e.data(), cap);
    m = nfc_reorder_compose(kNfc, e.data(), m, e.data() + cap, hist);
    std::string out(3 * (size_t)n + 4, '\0');
    out.resize(nfc_encode(e.data(), m, (uint8_t*)&out[0]));
    return out;
}

static std::string segmented(const uint8_t* s, uint32_t n) {
    std::string out;
    for (uint32_t i = 0, end; i < n; i = end) {
        end = nfc_segment_end(kNfc, s, i, n);
        uint32_t loc[32];
        uint8_t buf[4 * 32];
        const uint32_t m = nfc_decompose_text(kNfc, s, i, end, loc, 32);
        if (m <= 32) out.append((const char*)buf, nfc_encode(loc, nfc_reorder_compose(kNfc, loc, m, nullptr, nullptr), buf));
        else out += whole(s + i, end - i);
    }
    return out;
}

static void put(const std::string& s) {
    const uint32_t n = (uint32_t)s.size();
    std::fwrite(&n, 4, 1, stdout);
    std::fwrite(s.data(), 1, n, stdout);
}

int main(int argc, char** argv) {
    const bool nfc = argc > 1 && !std::strcmp(argv[1], "nfc");
    uint32_t len;
    while (std::fread(&len, 4, 1, stdin) == 1) {
        std::string text(len, '\0');
        if (len && std::fread(&text[0], 1, len, stdin) != len) return 2;
        const uint8_t* s = (const uint8_t*)text.data();
        if (nfc) { put(segmented(s, len)); put(whole(s, len)); }
        else split(s, len);
    }
    return 0;
}
