// Host build of the DeepSeek pre-tokenizer of smg_b200/csrc/bpe.cuh on the deepseek_tables.h classes, compiled with g++ so that
// tests/test_deepseek_host.py can compare exactly the code the kernel runs with live `tokenizers`.
//   test_deepseek_host split    stdin: records of (u32 little-endian byte length, UTF-8 bytes); three lines per record: "S <piece starts
//                               of the serial split>", "A <anchors>", "G <starts of the anchored split the GPU kernel does: from every
//                               anchor, replay the matcher up to the next anchor>"
//   test_deepseek_host classes  stdout: ds_class() of every code point U+0000 … U+10FFFF, one byte each (surrogates included)
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "bpe.cuh"
#include "deepseek_tables.h"

using namespace smgx;

static const UnicodeView kDs{kDsLo, kDsHi, kDsCls, kDsRanges};

static void print(const char* tag, const std::vector<uint32_t>& v) {
    std::fputs(tag, stdout);
    for (uint32_t x : v) std::printf(" %u", x);
    std::fputc('\n', stdout);
}

static void split(const uint8_t* s, uint32_t len) {
    std::vector<uint32_t> starts, anchors, seg;
    for (uint32_t i = 0; i < len; i = next_piece_deepseek(s, i, len, kDs)) starts.push_back(i);
    std::vector<uint8_t> is_anchor(len, 0);
    for (uint32_t i = 0; i < len; ++i)
        if ((s[i] & 0xC0) != 0x80 && is_anchor_deepseek(s, i, 0, nullptr, kDs)) { anchors.push_back(i); is_anchor[i] = 1; }
    for (uint32_t p : anchors)
        do { seg.push_back(p); p = next_piece_deepseek(s, p, len, kDs); } while (p < len && !is_anchor[p]);
    print("S", starts);
    print("A", anchors);
    print("G", seg);
}

int main(int argc, char** argv) {
    if (argc > 1 && !std::strcmp(argv[1], "classes")) {
        std::vector<uint8_t> out(0x110000);
        for (uint32_t cp = 0; cp < 0x110000; ++cp) out[cp] = ds_class(cp, kDs);
        std::fwrite(out.data(), 1, out.size(), stdout);
        return 0;
    }
    uint32_t len;
    while (std::fread(&len, 4, 1, stdin) == 1) {
        std::string text(len, '\0');
        if (len && std::fread(&text[0], 1, len, stdin) != len) return 2;
        split((const uint8_t*)text.data(), len);
    }
    return 0;
}
