// K1 — Unicode NFC as host+device functions, for tokenizer.json files whose normalizer is {"type": "NFC"} (Qwen2 and later).
//
// The reference normalizes through the `tokenizers` crate (HuggingFaceTokenizer::encode, crates/tokenizer/src/huggingface.rs), whose
// Unicode tables are older than Python's: nfc_tables.h is pinned to that behaviour by tools/gen_nfc_tables.py.
// NFC = full canonical decomposition, canonical ordering (a stable sort of every run of non-starters by combining class), then
// canonical composition (each character composes with the last starter unless a character of class 0 or of a class ≥ its own sits
// between them).  Compiles with g++ too (tests/cpp/test_qwen2_host.cpp runs exactly this code against `tokenizers`).
//
// Work is split at NFC-stable code points (nfc_stable): NFC never looks across the boundary before one, so the text between two of
// them is normalized on its own.  Code points are carried as entries `cp | ccc << 24`.
#pragma once
#include <cstdint>

#include "bpe.cuh"   // utf8_decode, SMGX_HD

namespace smgx {

struct NfcView {
    const uint32_t* ccc_cp; const uint8_t* ccc_val; uint32_t n_ccc;
    const uint32_t* dec_cp; const uint16_t* dec_off; const uint32_t* dec_data; uint32_t n_dec;
    const uint64_t* comp_key; const uint32_t* comp_val; uint32_t n_comp;
    const uint32_t* unst_lo; const uint32_t* unst_hi; uint32_t n_unst;
};

constexpr uint32_t kNfcCpMask = 0x1FFFFFu;
constexpr uint32_t kNfcSortSmall = 32;   // runs of non-starters up to this length are insertion-sorted, longer ones counting-sorted
constexpr uint32_t kHangulS = 0xAC00, kHangulL = 0x1100, kHangulV = 0x1161, kHangulT = 0x11A7;
constexpr uint32_t kHangulLCount = 19, kHangulVCount = 21, kHangulTCount = 28, kHangulNCount = 588, kHangulSCount = 11172;

template <class T>
SMGX_HD uint32_t nfc_lower_bound(const T* a, uint32_t n, T x) {   // first index with a[k] >= x
    uint32_t lo = 0, hi = n;
    while (lo < hi) {
        const uint32_t m = (lo + hi) >> 1;
        if (a[m] < x) lo = m + 1; else hi = m;
    }
    return lo;
}

SMGX_HD uint32_t nfc_ccc(const NfcView& v, uint32_t cp) {
    if (cp < 0x300) return 0;
    const uint32_t k = nfc_lower_bound(v.ccc_cp, v.n_ccc, cp);
    return k < v.n_ccc && v.ccc_cp[k] == cp ? v.ccc_val[k] : 0;
}

// NFC-stable: class 0, never the second half of a composition, its own NFC, and its decomposition starts with such a starter.
// Everything below U+0300 is stable (the generator asserts it), so ASCII and Latin-1 need no lookup.
SMGX_HD bool nfc_stable(const NfcView& v, uint32_t cp) {
    if (cp < 0x300) return true;
    const uint32_t k = nfc_lower_bound(v.unst_hi, v.n_unst, cp);   // first range with hi >= cp
    return !(k < v.n_unst && v.unst_lo[k] <= cp);
}

SMGX_HD uint32_t nfc_entry(const NfcView& v, uint32_t cp) { return cp | (nfc_ccc(v, cp) << 24); }

// Full canonical decomposition of cp as entries; returns the count (1 to 4; the generator asserts the bound).
SMGX_HD uint32_t nfc_decompose(const NfcView& v, uint32_t cp, uint32_t* out) {
    if (cp - kHangulS < kHangulSCount) {
        const uint32_t s = cp - kHangulS;
        out[0] = kHangulL + s / kHangulNCount;
        out[1] = kHangulV + (s % kHangulNCount) / kHangulTCount;
        if (s % kHangulTCount) { out[2] = kHangulT + s % kHangulTCount; return 3; }
        return 2;
    }
    if (cp >= 0xC0) {
        const uint32_t k = nfc_lower_bound(v.dec_cp, v.n_dec, cp);
        if (k < v.n_dec && v.dec_cp[k] == cp) {
            const uint32_t a = v.dec_off[k], b = v.dec_off[k + 1];
            for (uint32_t j = a; j < b; ++j) out[j - a] = nfc_entry(v, v.dec_data[j]);
            return b - a;
        }
    }
    out[0] = nfc_entry(v, cp);
    return 1;
}

// Primary composite of (a, b), or 0.
SMGX_HD uint32_t nfc_compose(const NfcView& v, uint32_t a, uint32_t b) {
    if (a - kHangulL < kHangulLCount && b - kHangulV < kHangulVCount) return kHangulS + ((a - kHangulL) * kHangulVCount + (b - kHangulV)) * kHangulTCount;
    if (a - kHangulS < kHangulSCount && (a - kHangulS) % kHangulTCount == 0 && b - kHangulT - 1 < kHangulTCount - 1) return a + (b - kHangulT);
    const uint64_t key = ((uint64_t)a << 21) | b;
    const uint32_t k = nfc_lower_bound(v.comp_key, v.n_comp, key);
    return k < v.n_comp && v.comp_key[k] == key ? v.comp_val[k] : 0;
}

// Stable sort of a run of non-starter entries by class.  Short runs: insertion sort in place.  Long runs (tmp and hist given):
// counting sort over the 256 classes through tmp — linear, exact at any length.
SMGX_HD void nfc_sort_run(uint32_t* e, uint32_t n, uint32_t* tmp, uint32_t* hist) {
    if (n <= kNfcSortSmall || tmp == nullptr) {
        for (uint32_t i = 1; i < n; ++i) {
            const uint32_t x = e[i];
            uint32_t j = i;
            while (j > 0 && (e[j - 1] >> 24) > (x >> 24)) { e[j] = e[j - 1]; --j; }
            e[j] = x;
        }
        return;
    }
    for (uint32_t c = 0; c < 256; ++c) hist[c] = 0;
    for (uint32_t i = 0; i < n; ++i) ++hist[e[i] >> 24];
    uint32_t run = 0;
    for (uint32_t c = 0; c < 256; ++c) { const uint32_t h = hist[c]; hist[c] = run; run += h; }
    for (uint32_t i = 0; i < n; ++i) tmp[hist[e[i] >> 24]++] = e[i];
    for (uint32_t i = 0; i < n; ++i) e[i] = tmp[i];
}

// Canonical ordering then canonical composition of the decomposed entries e[0..n), in place; returns the new count.
SMGX_HD uint32_t nfc_reorder_compose(const NfcView& v, uint32_t* e, uint32_t n, uint32_t* tmp, uint32_t* hist) {
    for (uint32_t i = 0; i < n;) {
        if ((e[i] >> 24) == 0) { ++i; continue; }
        uint32_t j = i + 1;
        while (j < n && (e[j] >> 24) != 0) ++j;
        if (j - i > 1) nfc_sort_run(e + i, j - i, tmp, hist);
        i = j;
    }
    // composition: `starter` = index of the last starter kept; `between` = a kept non-starter follows it, `last` = the class of the last one
    int64_t starter = -1;
    bool between = false;
    uint32_t last = 0, out = 0;
    for (uint32_t i = 0; i < n; ++i) {
        const uint32_t x = e[i], cc = x >> 24;
        if (starter >= 0 && !(between && last >= cc)) {
            const uint32_t r = nfc_compose(v, e[starter] & kNfcCpMask, x & kNfcCpMask);
            if (r) { e[starter] = r | (nfc_ccc(v, r) << 24); continue; }
        }
        if (cc == 0) { starter = out; between = false; }
        else { between = true; last = cc; }
        e[out++] = x;
    }
    return out;
}

// Decode s[i..end) (valid UTF-8) and decompose it into e[0..cap); returns the entry count, or cap + 1 when it does not fit.
SMGX_HD uint32_t nfc_decompose_text(const NfcView& v, const uint8_t* s, uint32_t i, uint32_t end, uint32_t* e, uint32_t cap) {
    uint32_t n = 0, d[4];
    while (i < end) {
        uint32_t l;
        const uint32_t cp = utf8_decode(s, i, end, l);
        i += l;
        const uint32_t k = nfc_decompose(v, cp, d);
        if (n + k > cap) return cap + 1;
        for (uint32_t j = 0; j < k; ++j) e[n + j] = d[j];
        n += k;
    }
    return n;
}

SMGX_HD uint32_t utf8_put(uint32_t cp, uint8_t* o) {
    if (cp < 0x80) { o[0] = (uint8_t)cp; return 1; }
    if (cp < 0x800) { o[0] = (uint8_t)(0xC0 | (cp >> 6)); o[1] = (uint8_t)(0x80 | (cp & 0x3F)); return 2; }
    if (cp < 0x10000) { o[0] = (uint8_t)(0xE0 | (cp >> 12)); o[1] = (uint8_t)(0x80 | ((cp >> 6) & 0x3F)); o[2] = (uint8_t)(0x80 | (cp & 0x3F)); return 3; }
    o[0] = (uint8_t)(0xF0 | (cp >> 18)); o[1] = (uint8_t)(0x80 | ((cp >> 12) & 0x3F)); o[2] = (uint8_t)(0x80 | ((cp >> 6) & 0x3F)); o[3] = (uint8_t)(0x80 | (cp & 0x3F));
    return 4;
}

// UTF-8 of the entries e[0..n) into o; returns the byte count (at most 3x the bytes the entries were decoded from).
SMGX_HD uint32_t nfc_encode(const uint32_t* e, uint32_t n, uint8_t* o) {
    uint32_t b = 0;
    for (uint32_t i = 0; i < n; ++i) b += utf8_put(e[i] & kNfcCpMask, o + b);
    return b;
}

// End of the NFC segment that starts at the lead byte i of s[..end): the next NFC-stable code point, or `end`.  `stop` (nullable)
// marks special-token bytes (value ≥ 2), which also end a segment: the text between two specials is normalized on its own.
SMGX_HD uint32_t nfc_segment_end(const NfcView& v, const uint8_t* s, uint32_t i, uint32_t end, const uint8_t* stop = nullptr) {
    uint32_t l;
    utf8_decode(s, i, end, l);
    uint32_t j = i + l;
    while (j < end) {
        if (stop != nullptr && stop[j] >= 2) break;
        const uint32_t cp = utf8_decode(s, j, end, l);
        if (nfc_stable(v, cp)) break;
        j += l;
    }
    return j;
}

}  // namespace smgx
