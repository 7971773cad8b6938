// K1 — SentencePiece-style BPE (Llama 2, Mistral, TinyLlama, CodeLlama): the ▁ normalization, the segmenter and the character-level
// symbolizer as host+device functions (tokenizer.cu runs them in kernels, tests/cpp/test_metaspace_host.cpp on the host).
//
// Two tokenizer.json shapes express the same idea, "a space is ▁ (U+2581) and a stretch of text starts with ▁":
//   legacy     normalizer Sequence[Prepend("▁"), Replace(" " → "▁")], no pre-tokenizer: every non-empty stretch between added tokens
//              gets a ▁ in front, even one that already starts with a space;
//   metaspace  no normalizer, pre_tokenizer Metaspace(replacement "▁", prepend_scheme, split): spaces become ▁ and then a ▁ is prepended
//              unless the stretch already starts with one; prepend_scheme "first" only does so for the stretch at offset 0 of the
//              request, "never" never.  split = true cuts the stretch before every ▁ (MergedWithNext).
// The BPE "word" is then a whole stretch.  The GPU cuts it before every ▁ that follows another character (split = false), or before
// every ▁ (split = true), and merges the pieces independently.  For split = false this is exact when no merge (a, b) has `a` ending in
// a character other than ▁ (or being a byte token) and `b` starting with ▁ — Tokenizer::build checks that (DESIGN §4c).
// Initial symbols are code points looked up in the vocabulary; one that is not there becomes the <0xXX> tokens of its bytes.
#pragma once
#include <cstdint>

#include "bpe.cuh"

namespace smgx {

enum : uint32_t { MS_PREPEND_NEVER = 0, MS_PREPEND_FIRST = 1, MS_PREPEND_ALWAYS = 2, MS_PREPEND_LEGACY = 3 /* Prepend normalizer */ };
struct MetaspaceMode {
    uint32_t on;        // 0: not a SentencePiece-style tokenizer
    uint32_t prepend;   // MS_PREPEND_*
    uint32_t split;     // 1: a piece starts at every ▁
};
constexpr uint32_t kMsInvalid = 0xFFFFFFFFu;

SMGX_HD bool is_metaspace_at(const uint8_t* s, uint32_t i) {   // ▁ = E2 96 81; valid UTF-8, so a lead E2 has its two continuation bytes
    return s[i] == 0xE2 && s[i + 1] == 0x96 && s[i + 2] == 0x81;
}

// Normalization, per byte of the raw text.  flags as in tokenizer.cu: < 2 ordinary, 2 first byte of a special, 3 inside one.
// Is a ▁ written in front of raw byte i (the first byte of a non-empty stretch)?
SMGX_HD bool ms_prepends(const MetaspaceMode& m, const uint8_t* s, const uint8_t* flags, uint32_t i, uint32_t beg) {
    if (flags[i] >= 2 || !(i == beg || flags[i - 1] >= 2)) return false;
    if (m.prepend == MS_PREPEND_LEGACY) return true;
    if (m.prepend == MS_PREPEND_NEVER || (m.prepend == MS_PREPEND_FIRST && i != beg)) return false;
    return !(s[i] == ' ' || is_metaspace_at(s, i));
}
// Bytes of normalized text that raw byte i becomes: a special's byte stays, a space is ▁, plus the prepended ▁.  At most 6.
SMGX_HD uint32_t ms_out_len(const MetaspaceMode& m, const uint8_t* s, const uint8_t* flags, uint32_t i, uint32_t beg) {
    if (flags[i] >= 2) return 1;
    return (ms_prepends(m, s, flags, i, beg) ? 3u : 0u) + (s[i] == ' ' ? 3u : 1u);
}
SMGX_HD uint32_t ms_out_write(const MetaspaceMode& m, const uint8_t* s, const uint8_t* flags, uint32_t i, uint32_t beg, uint8_t* out) {
    uint32_t k = 0;
    if (flags[i] < 2) {
        if (ms_prepends(m, s, flags, i, beg)) { out[0] = 0xE2; out[1] = 0x96; out[2] = 0x81; k = 3; }
        if (s[i] == ' ') { out[k] = 0xE2; out[k + 1] = 0x96; out[k + 2] = 0x81; return k + 3; }
    }
    out[k] = s[i];
    return k + 1;
}

// Segmenter, on the normalized text: does a piece start at lead byte i (flags[i] < 2)?  At the stretch start, and before a ▁ that follows
// another character of the stretch (split = false) or before every ▁ (split = true).
SMGX_HD bool ms_piece_start(const uint8_t* s, const uint8_t* flags, uint32_t i, uint32_t beg, uint32_t split) {
    if (i == beg || flags[i - 1] >= 2) return true;
    if (!is_metaspace_at(s, i)) return false;
    if (split) return true;
    return !(i - beg >= 3 && s[i - 1] == 0x81 && s[i - 2] == 0x96 && s[i - 3] == 0xE2);   // the character before is not ▁
}

// Symbolizer: the initial symbols of the code point at lead byte i of s[..n).  Its vocabulary id in out[0], or (byte fallback) the <0xXX>
// token of every byte in out[0..len); the other slots get kMsInvalid.  Returns the code point's byte length.
SMGX_HD uint32_t ms_symbolize(const BpeView& v, const uint8_t* s, uint32_t i, uint32_t n, uint32_t* out, uint32_t* n_sym) {
    uint32_t len, id;
    utf8_decode(s, i, n, len);
    if (piece_lookup(v, s + i, len, id)) {
        out[0] = id;
        for (uint32_t k = 1; k < len; ++k) out[k] = kMsInvalid;
        *n_sym = 1;
    } else {
        for (uint32_t k = 0; k < len; ++k) out[k] = v.byte_token[s[i + k]];
        *n_sym = len;
    }
    return len;
}

}  // namespace smgx
