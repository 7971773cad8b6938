// Host build of the GPT-2 (r50k) pre-tokenizer of smg_b200/csrc/bpe.cuh: next_piece_r50k and the r50k anchor rule, compiled with g++
// so that tests/test_r50k_splitter.py can compare them with the regex on the CPU.
//
// stdin: records of (u32 little-endian byte length, UTF-8 bytes).  stdout, three lines per record:
//   S <starts>   piece starts of the serial split (next_piece_r50k from byte 0 to the end)
//   A <anchors>  bytes that is_anchor_r50k marks (every lead byte is tested)
//   G <starts>   piece starts of the anchored split the GPU kernel does: from every anchor, replay the matcher up to the next anchor
#include <cstdint>
#include <cstdio>
#include <string>
#include <vector>

#include "bpe.cuh"
#include "unicode_tables.h"

using namespace smgx;

static void print(const char* tag, const std::vector<uint32_t>& v) {
    std::fputs(tag, stdout);
    for (uint32_t x : v) std::printf(" %u", x);
    std::fputc('\n', stdout);
}

int main() {
    const UnicodeView u{kUniLo, kUniHi, kUniCls, kUniRanges};
    uint32_t len;
    while (std::fread(&len, 4, 1, stdin) == 1) {
        std::string text(len, '\0');
        if (len && std::fread(&text[0], 1, len, stdin) != len) return 2;
        const uint8_t* s = (const uint8_t*)text.data();
        std::vector<uint32_t> starts, anchors, seg;
        for (uint32_t i = 0; i < len;) {
            starts.push_back(i);
            const uint32_t e = next_piece_r50k(s, i, len, u);
            if (e <= i) return 3;   // the matcher must make progress
            i = e;
        }
        std::vector<uint8_t> is_anchor(len, 0);
        for (uint32_t i = 0; i < len; ++i)
            if ((s[i] & 0xC0) != 0x80 && is_anchor_r50k(s, i, 0, nullptr, u)) { anchors.push_back(i); is_anchor[i] = 1; }
        for (uint32_t a : anchors) {
            uint32_t p = a;
            for (;;) {
                seg.push_back(p);
                p = next_piece_r50k(s, p, len, u);
                if (p >= len || is_anchor[p]) break;
            }
        }
        print("S", starts);
        print("A", anchors);
        print("G", seg);
    }
    return 0;
}
