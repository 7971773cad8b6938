// K1 — tokenize: the cl100k and GPT-2 (r50k) pre-tokenizers and tiktoken-style byte-pair merge as host+device functions.
//
// Replaces, token for token, what the reference gets from the un-vendored crate tiktoken-rs through
//   TiktokenTokenizer::encode → CoreBPE::encode_with_special_tokens   crates/tokenizer/src/tiktoken.rs:444-462
// with the pattern CL100K_BASE_PATTERN (tiktoken.rs:28):
//   (?i:'s|'t|'re|'ve|'m|'ll|'d) | [^\r\n\p{L}\p{N}]?\p{L}+ | \p{N}{1,3} | ?[^\s\p{L}\p{N}]+[\r\n]* | \s*[\r\n]+ | \s+(?!\S) | \s+
// or with the GPT-2 pattern of r50k_base / p50k_base / p50k_edit (next_piece_r50k below).
// Each regex is compiled by hand into a next_piece_*() function: leftmost-first alternation, greedy quantifiers and the one
// backtracking look-ahead are resolved analytically (see the comments at each alternative).
#pragma once
#include <cstdint>

#include "xxh3.cuh"  // SMGX_HD

namespace smgx {

enum : uint8_t { CH_OTHER = 0, CH_LETTER = 1, CH_NUMBER = 2, CH_SPACE = 3 /* White_Space */ };

struct UnicodeView {
    const uint32_t* lo;   // sorted range starts
    const uint32_t* hi;
    const uint8_t* cls;
    uint32_t n;
};

// UTF-8 decode at s[i] (input is valid UTF-8, as `&str` guarantees in the reference); len = bytes consumed.
SMGX_HD uint32_t utf8_decode(const uint8_t* s, uint32_t i, uint32_t n, uint32_t& len) {
    uint32_t c = s[i];
    if (c < 0x80) { len = 1; return c; }
    if ((c >> 5) == 0x6 && i + 1 < n) { len = 2; return ((c & 0x1F) << 6) | (s[i + 1] & 0x3F); }
    if ((c >> 4) == 0xE && i + 2 < n) { len = 3; return ((c & 0x0F) << 12) | ((s[i + 1] & 0x3F) << 6) | (s[i + 2] & 0x3F); }
    if ((c >> 3) == 0x1E && i + 3 < n) { len = 4; return ((c & 0x07) << 18) | ((s[i + 1] & 0x3F) << 12) | ((s[i + 2] & 0x3F) << 6) | (s[i + 3] & 0x3F); }
    len = 1;
    return 0xFFFD;
}

SMGX_HD uint8_t char_class(uint32_t cp, const UnicodeView& u) {
    if (cp < 0x80) {
        if ((cp >= 'a' && cp <= 'z') || (cp >= 'A' && cp <= 'Z')) return CH_LETTER;
        if (cp >= '0' && cp <= '9') return CH_NUMBER;
        if (cp == ' ' || (cp >= 0x09 && cp <= 0x0D)) return CH_SPACE;
        return CH_OTHER;
    }
    uint32_t a = 0, b = u.n;   // first range with hi >= cp
    while (a < b) {
        uint32_t m = (a + b) >> 1;
        if (u.hi[m] < cp) a = m + 1; else b = m;
    }
    if (a < u.n && u.lo[a] <= cp) return u.cls[a];
    return CH_OTHER;
}
SMGX_HD bool is_newline(uint32_t cp) { return cp == '\n' || cp == '\r'; }

// End (byte index) of the regex match that starts at byte i of s[0..n).  i < n and i is not a slice end.
// tiktoken runs the regex only on the ordinary text between two special tokens; `stop` (nullable) marks the first byte of
// every special with the value 2, and such a byte acts as the end of the string (for the run scans and for `(?!\S)`).
// kDigits is the longest digit run of alternative 3: \p{N}{1,3} in cl100k / Llama 3, \p{N} in Qwen2 (next_piece_qwen2 below).
template <int kDigits>
SMGX_HD uint32_t next_piece_llama(const uint8_t* s, uint32_t i, uint32_t n, const UnicodeView& u, const uint8_t* stop) {
#define SMGX_AT_END(j) ((j) >= n || (stop != nullptr && stop[(j)] == 2))
    uint32_t len0;
    const uint32_t cp0 = utf8_decode(s, i, n, len0);
    const uint8_t cls0 = char_class(cp0, u);

    // 1. (?i:'s|'t|'re|'ve|'m|'ll|'d) — Unicode-aware case folding adds U+017F (ſ) for 's'
    if (cp0 == '\'' && !SMGX_AT_END(i + 1)) {
        const uint32_t c1 = s[i + 1] | 0x20;
        if (s[i + 1] < 0x80) {
            if (c1 == 's' || c1 == 't' || c1 == 'm' || c1 == 'd') return i + 2;
            if (!SMGX_AT_END(i + 2) && s[i + 2] < 0x80) {
                const uint32_t c2 = s[i + 2] | 0x20;
                if ((c1 == 'r' && c2 == 'e') || (c1 == 'v' && c2 == 'e') || (c1 == 'l' && c2 == 'l')) return i + 3;
            }
        } else if (i + 2 < n && s[i + 1] == 0xC5 && s[i + 2] == 0xBF) {
            return i + 3;  // 'ſ
        }
    }
    // 2. [^\r\n\p{L}\p{N}]?\p{L}+   — the optional char is taken only when a letter follows it (otherwise the
    //    alternative can only match with the optional empty, which needs a letter at i)
    {
        uint32_t j = i;
        bool ok = cls0 == CH_LETTER;
        if (!ok && cls0 != CH_NUMBER && !is_newline(cp0)) {
            uint32_t k = i + len0;
            if (!SMGX_AT_END(k)) {
                uint32_t l1;
                uint32_t cp1 = utf8_decode(s, k, n, l1);
                if (char_class(cp1, u) == CH_LETTER) { j = k; ok = true; }
            }
        }
        if (ok) {
            while (!SMGX_AT_END(j)) {
                uint32_t l;
                uint32_t cp = utf8_decode(s, j, n, l);
                if (char_class(cp, u) != CH_LETTER) break;
                j += l;
            }
            return j;
        }
    }
    // 3. \p{N}{1,3}  (Qwen2: \p{N})
    if (cls0 == CH_NUMBER) {
        uint32_t j = i + len0;
        for (int c = 1; c < kDigits && !SMGX_AT_END(j); ++c) {
            uint32_t l;
            uint32_t cp = utf8_decode(s, j, n, l);
            if (char_class(cp, u) != CH_NUMBER) break;
            j += l;
        }
        return j;
    }
    // 4.  ?[^\s\p{L}\p{N}]+[\r\n]*
    {
        uint32_t j = i;
        bool ok = cls0 == CH_OTHER;
        if (!ok && cp0 == ' ' && !SMGX_AT_END(i + 1)) {
            uint32_t l1;
            uint32_t cp1 = utf8_decode(s, i + 1, n, l1);
            if (char_class(cp1, u) == CH_OTHER) { j = i + 1; ok = true; }
        }
        if (ok) {
            while (!SMGX_AT_END(j)) {
                uint32_t l;
                uint32_t cp = utf8_decode(s, j, n, l);
                if (char_class(cp, u) != CH_OTHER) break;
                j += l;
            }
            while (!SMGX_AT_END(j) && (s[j] == '\n' || s[j] == '\r')) ++j;
            return j;
        }
    }
    // 5-7. whitespace run starting at i (cls0 == CH_SPACE)
    uint32_t j = i, last_nl_end = 0, last_start = i, count = 0;
    while (!SMGX_AT_END(j)) {
        uint32_t l;
        uint32_t cp = utf8_decode(s, j, n, l);
        if (char_class(cp, u) != CH_SPACE) break;
        last_start = j;
        j += l;
        ++count;
        if (is_newline(cp)) last_nl_end = j;
    }
    if (last_nl_end) return last_nl_end;   // 5. \s*[\r\n]+  : greedy \s* backtracks to the last newline of the run
    if (SMGX_AT_END(j)) return j;          // 6. \s+(?!\S)   : run reaches the end of the (slice of) text
    if (count >= 2) return last_start;     // 6.             : give back one char so that whitespace follows
    return j;                              // 7. \s+
#undef SMGX_AT_END
}
SMGX_HD uint32_t next_piece_cl100k(const uint8_t* s, uint32_t i, uint32_t n, const UnicodeView& u, const uint8_t* stop = nullptr) {
    return next_piece_llama<3>(s, i, n, u, stop);
}

// ---- Qwen2 pre-tokenizer -------------------------------------------------------------------------------------------
// The Split regex of the Qwen2 / Qwen2.5 / Qwen3 tokenizer.json files: the cl100k pattern with \p{N} in place of \p{N}{1,3},
//   (?i:'s|'t|'re|'ve|'m|'ll|'d) | [^\r\n\p{L}\p{N}]?\p{L}+ | \p{N} | ?[^\s\p{L}\p{N}]+[\r\n]* | \s*[\r\n]+ | \s+(?!\S) | \s+
// so every digit is a piece of its own.  Anchor rule: cl100k's, except that every digit and the character after every digit start a
// piece (no other alternative can take a digit).
SMGX_HD uint32_t next_piece_qwen2(const uint8_t* s, uint32_t i, uint32_t n, const UnicodeView& u, const uint8_t* stop = nullptr) {
    return next_piece_llama<1>(s, i, n, u, stop);
}
SMGX_HD bool qwen2_anchor_rule(uint8_t pc, uint8_t c) { return (pc == CH_LETTER && c != CH_LETTER) || c == CH_NUMBER || pc == CH_NUMBER; }

// ---- GPT-2 / r50k pre-tokenizer ------------------------------------------------------------------------------------
// tiktoken's r50k_pat_str (r50k_base, p50k_base, p50k_edit) and `tokenizers`' ByteLevel(use_regex = true), in the form
//   's|'t|'re|'ve|'m|'ll|'d | ?\p{L}+ | ?\p{N}+ | ?[^\s\p{L}\p{N}]+ | \s+(?!\S) | \s+
// Same contract as next_piece_cl100k.  Differences that matter: contractions are case-sensitive, digit runs are unbounded,
// only U+0020 may lead a run, and there is no newline rule.
enum class Pretok : uint8_t { Cl100k = 0, R50k = 1, Qwen2 = 2, DeepSeek = 4 };

SMGX_HD bool is_contraction_tail(uint8_t b) {   // second byte of 's 't 'm 'd 're 've 'll
    return b == 's' || b == 't' || b == 'm' || b == 'd' || b == 'r' || b == 'v' || b == 'l';
}

SMGX_HD uint32_t next_piece_r50k(const uint8_t* s, uint32_t i, uint32_t n, const UnicodeView& u, const uint8_t* stop = nullptr) {
#define SMGX_AT_END(j) ((j) >= n || (stop != nullptr && stop[(j)] == 2))
    uint32_t len0;
    const uint32_t cp0 = utf8_decode(s, i, n, len0);
    const uint8_t cls0 = char_class(cp0, u);

    // 1. 's|'t|'re|'ve|'m|'ll|'d   (case-sensitive; the continuation bytes are ASCII, so bytes compare as characters)
    if (cp0 == '\'' && !SMGX_AT_END(i + 1)) {
        const uint8_t b1 = s[i + 1];
        if (b1 == 's' || b1 == 't' || b1 == 'm' || b1 == 'd') return i + 2;
        if ((b1 == 'r' || b1 == 'v' || b1 == 'l') && !SMGX_AT_END(i + 2)) {
            const uint8_t b2 = s[i + 2];
            if (b1 == 'l' ? b2 == 'l' : b2 == 'e') return i + 3;
        }
    }
    // 2-4.  ?\p{L}+ |  ?\p{N}+ |  ?[^\s\p{L}\p{N}]+   — the three alternatives start with disjoint classes, so together they are
    //      "a run of one non-space class, optionally led by one U+0020".  The space is taken only when a non-space follows it;
    //      otherwise none of the three can match at i and the whitespace alternatives decide.
    {
        uint32_t j = i;
        uint8_t rc = cls0;
        if (cp0 == ' ' && !SMGX_AT_END(i + 1)) {
            uint32_t l1;
            const uint8_t c1 = char_class(utf8_decode(s, i + 1, n, l1), u);
            if (c1 != CH_SPACE) { j = i + 1; rc = c1; }
        }
        if (rc != CH_SPACE) {
            while (!SMGX_AT_END(j)) {
                uint32_t l;
                const uint32_t cp = utf8_decode(s, j, n, l);
                if (char_class(cp, u) != rc) break;
                j += l;
            }
            return j;
        }
    }
    // 5-6. whitespace run starting at i (cls0 == CH_SPACE)
    uint32_t j = i, last_start = i, count = 0;
    while (!SMGX_AT_END(j)) {
        uint32_t l;
        const uint32_t cp = utf8_decode(s, j, n, l);
        if (char_class(cp, u) != CH_SPACE) break;
        last_start = j;
        j += l;
        ++count;
    }
    if (SMGX_AT_END(j)) return j;          // 5. \s+(?!\S) : run reaches the end of the (slice of) text
    if (count >= 2) return last_start;     // 5.            : give back one char so that whitespace follows
    return j;                              // 6. \s+        : a single whitespace char before a non-space
#undef SMGX_AT_END
}

// Anchor rule of the r50k pattern: a piece certainly starts at p when the character before p is not whitespace and its class differs
// from the class at p — unless that character is ' and the byte at p can continue a contraction.  `pc`/`pb` are the class and the
// last byte of the previous character, `c`/`b` the class and the first byte of the character at p.  (Why it holds: DESIGN §4c.)
SMGX_HD bool r50k_anchor_rule(uint8_t pc, uint8_t pb, uint8_t c, uint8_t b) {
    if (pc == CH_SPACE || pc == c) return false;
    return !(pb == '\'' && is_contraction_tail(b));
}

SMGX_HD uint32_t prev_cp(const uint8_t* s, uint32_t i, uint32_t lo) {   // code point ending right before byte i
    uint32_t j = i - 1;
    while (j > lo && (s[j] & 0xC0) == 0x80) --j;
    uint32_t l;
    return utf8_decode(s, j, i, l);
}

// Is byte i of the request s[beg..) (a lead byte, not inside a special) an r50k anchor?  `flags` (nullable) marks specials as in
// next_piece_*: the byte after a special is an anchor, as is the request start.
SMGX_HD bool is_anchor_r50k(const uint8_t* s, uint32_t i, uint32_t beg, const uint8_t* flags, const UnicodeView& u) {
    if (i == beg) return true;
    if (flags != nullptr && flags[i - 1] >= 2) return true;
    uint32_t l;
    const uint8_t c = char_class(utf8_decode(s, i, i + 4, l), u);   // valid UTF-8: a lead byte's continuation bytes exist
    const uint8_t pc = char_class(prev_cp(s, i, beg), u);
    return r50k_anchor_rule(pc, s[i - 1], c, s[i]);
}
// Same for the Qwen2 pattern (qwen2_anchor_rule).
SMGX_HD bool is_anchor_qwen2(const uint8_t* s, uint32_t i, uint32_t beg, const uint8_t* flags, const UnicodeView& u) {
    if (i == beg) return true;
    if (flags != nullptr && flags[i - 1] >= 2) return true;
    uint32_t l;
    const uint8_t c = char_class(utf8_decode(s, i, i + 4, l), u);
    const uint8_t pc = char_class(prev_cp(s, i, beg), u);
    return qwen2_anchor_rule(pc, c);
}

// ---- DeepSeek pre-tokenizer ----------------------------------------------------------------------------------------
// The tokenizer.json of DeepSeek V2 / V2.5 / Coder-V2 / V3 / V3.1 / R1 chains three Isolated Splits; each runs on every piece the one
// before produced, a piece's end is the end of the string for the next regex, and unmatched gaps are pieces too:
//   1. \p{N}{1,3}             digit runs, cut in triples counted from the start of the run
//   2. [一-龥぀-ゟ゠-ヿ]+         kana/CJK runs (U+4E00-U+9FA5, U+3040-U+30FF); the generator asserts that no digit lies in them
//   3. [!"#$%&'()*+,\-./:;<=>?@\[\\\]^_`{|}~][A-Za-z]+ | [^\r\n\p{L}\p{P}\p{S}]?[\p{L}\p{M}]+ | ?[\p{P}\p{S}]+[\r\n]* | \s*[\r\n]+ |
//      \s+(?!\S) | \s+         on each kana/CJK run and on each stretch between digit and kana/CJK runs ("stage pieces")
// The classes are those of `tokenizers` (Oniguruma), from deepseek_tables.h, not those of unicode_tables.h.
enum : uint8_t { DS_OTHER = 0, DS_L = 1, DS_M = 2, DS_N = 3, DS_P = 4, DS_S = 5, DS_WS = 6, DS_KANA = 8 /* flag */ };
constexpr uint8_t kDsEnd = 0xFF;

SMGX_HD uint8_t ds_class(uint32_t cp, const UnicodeView& u) {   // u: the deepseek_tables.h ranges
    if (cp < 0x80) {
        if ((cp | 0x20) >= 'a' && (cp | 0x20) <= 'z') return DS_L;
        if (cp >= '0' && cp <= '9') return DS_N;
        if (cp == ' ' || (cp >= 0x09 && cp <= 0x0D)) return DS_WS;
        if (cp == '$' || cp == '+' || (cp >= '<' && cp <= '>') || cp == '^' || cp == '`' || cp == '|' || cp == '~') return DS_S;
        return cp >= 0x21 && cp <= 0x7E ? DS_P : DS_OTHER;
    }
    uint32_t a = 0, b = u.n;
    while (a < b) {
        uint32_t m = (a + b) >> 1;
        if (u.hi[m] < cp) a = m + 1; else b = m;
    }
    return a < u.n && u.lo[a] <= cp ? u.cls[a] : (uint8_t)DS_OTHER;
}
SMGX_HD bool ds_letter_or_mark(uint8_t c) { return c == DS_L || c == DS_M; }   // c without the kana flag
SMGX_HD bool ds_punct_or_symbol(uint8_t c) { return c == DS_P || c == DS_S; }
SMGX_HD bool is_ascii_letter(uint8_t b) { return (b | 0x20) >= 'a' && (b | 0x20) <= 'z'; }
// Class (kana flag dropped) of a character `c` (with its flag) seen from a stage piece of zone `z` (DS_KANA or 0), or kDsEnd when the
// character ends that piece: a digit, or a character of the other zone.
SMGX_HD uint8_t ds_stage_class(uint8_t c, uint8_t z) { return (c == DS_N || (c & DS_KANA) != z) ? kDsEnd : (uint8_t)(c & 7); }
// ds_stage_class and length l of the character at byte j of s[0..n); kDsEnd at n and at a special's first byte (`stop` as in
// next_piece_llama).
SMGX_HD uint8_t ds_at(const uint8_t* s, uint32_t j, uint32_t n, const UnicodeView& u, const uint8_t* stop, uint8_t z, uint32_t& l) {
    if (j >= n || (stop != nullptr && stop[j] == 2)) { l = 0; return kDsEnd; }
    return ds_stage_class(ds_class(utf8_decode(s, j, n, l), u), z);
}

// Same contract as next_piece_cl100k, for the whole chain: i is a piece start (a digit at i starts a triple).
SMGX_HD uint32_t next_piece_deepseek(const uint8_t* s, uint32_t i, uint32_t n, const UnicodeView& u, const uint8_t* stop = nullptr) {
#define SMGX_AT_END(j) ((j) >= n || (stop != nullptr && stop[(j)] == 2))
#define DS_AT(j, l) ds_at(s, (j), n, u, stop, c0 & DS_KANA, (l))
    uint32_t len0;
    const uint32_t cp0 = utf8_decode(s, i, n, len0);
    const uint8_t c0 = ds_class(cp0, u);
    uint32_t l;
    // Split 1: \p{N}{1,3}
    if (c0 == DS_N) {
        uint32_t j = i + len0;
        for (int c = 1; c < 3 && !SMGX_AT_END(j); ++c) {
            if (ds_class(utf8_decode(s, j, n, l), u) != DS_N) break;
            j += l;
        }
        return j;
    }
    // Split 3 inside the stage piece (kana/CJK run or the text between runs)
    const uint8_t c = c0 & 7;
    // 1. [ASCII punctuation][A-Za-z]+
    if (cp0 < 0x80 && ds_punct_or_symbol(c)) {
        uint32_t j = i + 1;
        while (!SMGX_AT_END(j) && is_ascii_letter(s[j])) ++j;
        if (j > i + 1) return j;
    }
    // 2. [^\r\n\p{L}\p{P}\p{S}]?[\p{L}\p{M}]+  — the optional char is taken only when a letter or mark follows it
    {
        uint32_t j = i;
        bool ok = ds_letter_or_mark(c);
        if (!ok && !ds_punct_or_symbol(c) && !is_newline(cp0) && ds_letter_or_mark(DS_AT(i + len0, l))) { j = i + len0; ok = true; }
        if (ok) {
            while (ds_letter_or_mark(DS_AT(j, l))) j += l;
            return j;
        }
    }
    // 3.  ?[\p{P}\p{S}]+[\r\n]*
    {
        uint32_t j = i;
        bool ok = ds_punct_or_symbol(c);
        if (!ok && cp0 == ' ' && ds_punct_or_symbol(DS_AT(i + 1, l))) { j = i + 1; ok = true; }
        if (ok) {
            while (ds_punct_or_symbol(DS_AT(j, l))) j += l;
            while (DS_AT(j, l) == DS_WS && (s[j] == '\n' || s[j] == '\r')) ++j;
            return j;
        }
    }
    // 4-6. whitespace run starting at i
    if (c == DS_WS) {
        uint32_t j = i, last_nl_end = 0, last_start = i, count = 0;
        while (DS_AT(j, l) == DS_WS) {
            last_start = j;
            const bool nl = s[j] == '\n' || s[j] == '\r';
            j += l;
            ++count;
            if (nl) last_nl_end = j;
        }
        if (last_nl_end) return last_nl_end;   // 4. \s*[\r\n]+
        if (DS_AT(j, l) == kDsEnd) return j;      // 5. \s+(?!\S): the run reaches the end of the stage piece
        if (count >= 2) return last_start;     // 5. give back one char so that whitespace follows
        return j;                              // 6. \s+
    }
    // no alternative matches at i (an "other" character not followed by a letter or mark): the gap runs up to the next character
    // where one does
    uint32_t j = i + len0;
    for (uint32_t lj; DS_AT(j, lj) == DS_OTHER && !ds_letter_or_mark(DS_AT(j + lj, l)); j += lj) {}
    return j;
#undef SMGX_AT_END
#undef DS_AT
}
// Anchor rule (DESIGN §4c): a piece certainly starts at the first character of every digit run and every kana/CJK run, at the first
// character after either, and at every character that is not a letter or mark after one that is.  pc / c: classes with the kana flag.
SMGX_HD bool deepseek_anchor_rule(uint8_t pc, uint8_t c) {
    return (c == DS_N) != (pc == DS_N) || (c & DS_KANA) != (pc & DS_KANA) || (ds_letter_or_mark(pc & 7) && !ds_letter_or_mark(c & 7));
}
// Is byte i of the request s[beg..) an anchor?  Same contract as is_anchor_r50k.
SMGX_HD bool is_anchor_deepseek(const uint8_t* s, uint32_t i, uint32_t beg, const uint8_t* flags, const UnicodeView& u) {
    if (i == beg) return true;
    if (flags != nullptr && flags[i - 1] >= 2) return true;
    uint32_t l;
    const uint8_t c = ds_class(utf8_decode(s, i, i + 4, l), u);
    const uint8_t pc = ds_class(prev_cp(s, i, beg), u);
    return deepseek_anchor_rule(pc, c);
}

// ---- vocabulary tables ---------------------------------------------------------------------------------------
struct PairSlot { uint64_t key; uint32_t rank; uint32_t id; };          // key = left_id << 32 | right_id ; empty = ~0
struct PieceSlot { uint64_t hash; uint32_t id; uint32_t len; uint32_t off; uint32_t pad; };  // hash 0 = empty
struct SpecialTok { uint32_t off, len, id, pad; };

struct BpeView {
    const uint32_t* byte_token;   // [256] id of each single-byte token
    const PairSlot* pairs;
    uint32_t pair_mask;
    const PieceSlot* pieces;
    uint32_t piece_mask;
    const uint8_t* blob;          // token bytes (piece verification) + special strings
    uint32_t max_token_len;
    const SpecialTok* specials;
    uint32_t n_special;
    uint32_t special_first[8];    // bitmap of first bytes of special strings
    uint32_t whole_piece;         // 1: a piece that is a vocabulary entry becomes that token without merging (tiktoken; HF ignore_merges)
    UnicodeView uni;
};

constexpr uint64_t kPairEmpty = ~0ULL;
constexpr uint32_t kRankMax = 0xFFFFFFFFu;

SMGX_HD uint64_t mix64(uint64_t x) {
    x ^= x >> 33; x *= 0xFF51AFD7ED558CCDULL; x ^= x >> 33; x *= 0xC4CEB9FE1A85EC53ULL; x ^= x >> 33;
    return x;
}
SMGX_HD uint64_t bytes_hash(const uint8_t* p, uint32_t n) {
    uint64_t h = 0xCBF29CE484222325ULL;
    for (uint32_t i = 0; i < n; ++i) { h ^= p[i]; h *= 0x100000001B3ULL; }
    h = mix64(h ^ n);
    return h ? h : 1;
}
// rank + merged id of the adjacent pair (l, r); rank kRankMax when bytes(l)+bytes(r) is not a vocab entry
SMGX_HD uint64_t pair_lookup(const BpeView& v, uint32_t l, uint32_t r) {
    const uint64_t key = ((uint64_t)l << 32) | r;
    uint32_t h = (uint32_t)(mix64(key) >> 32) & v.pair_mask;
    for (;;) {
        const PairSlot s = v.pairs[h];
        if (s.key == key) return ((uint64_t)s.rank << 32) | s.id;
        if (s.key == kPairEmpty) return ((uint64_t)kRankMax << 32);
        h = (h + 1) & v.pair_mask;
    }
}
// `self.encoder.get(piece)` — whole piece is one vocab entry?
SMGX_HD bool piece_lookup(const BpeView& v, const uint8_t* p, uint32_t n, uint32_t& id) {
    if (n > v.max_token_len) return false;
    const uint64_t hsh = bytes_hash(p, n);
    uint32_t h = (uint32_t)(hsh >> 32) & v.piece_mask;
    for (;;) {
        const PieceSlot s = v.pieces[h];
        if (s.hash == 0) return false;
        if (s.hash == hsh && s.len == n) {
            bool eq = true;
            for (uint32_t i = 0; i < n; ++i) if (v.blob[s.off + i] != p[i]) { eq = false; break; }
            if (eq) { id = s.id; return true; }
        }
        h = (h + 1) & v.piece_mask;
    }
}

// The merge loop of byte_pair_merge on symbols already in ids[0..n) (SentencePiece-style BPE: code points and byte-fallback tokens).
SMGX_HD uint32_t merge_symbols(const BpeView& v, uint32_t* ids, uint32_t n, uint64_t* rk) {
    if (n < 2) return n;
    for (uint32_t i = 0; i + 1 < n; ++i) rk[i] = pair_lookup(v, ids[i], ids[i + 1]);
    uint32_t m = n;
    for (;;) {
        uint32_t best = kRankMax, bi = 0;
        for (uint32_t i = 0; i + 1 < m; ++i) {       // leftmost minimum (strict <)
            uint32_t r = (uint32_t)(rk[i] >> 32);
            if (r < best) { best = r; bi = i; }
        }
        if (best == kRankMax) break;
        ids[bi] = (uint32_t)rk[bi];
        for (uint32_t i = bi + 1; i + 1 < m; ++i) { ids[i] = ids[i + 1]; rk[i] = rk[i + 1]; }
        --m;
        rk[bi] = (bi + 1 < m) ? pair_lookup(v, ids[bi], ids[bi + 1]) : ((uint64_t)kRankMax << 32);
        if (bi > 0) rk[bi - 1] = pair_lookup(v, ids[bi - 1], ids[bi]);
    }
    return m;
}
// tiktoken `_byte_pair_merge` over token ids: ids[0..n) start as the single-byte tokens of the piece, rk[i] packs
// (rank, merged id) of the pair (ids[i], ids[i+1]).  Returns the number of tokens left in ids[].
SMGX_HD uint32_t byte_pair_merge(const BpeView& v, const uint8_t* p, uint32_t n, uint32_t* ids, uint64_t* rk) {
    for (uint32_t i = 0; i < n; ++i) ids[i] = v.byte_token[p[i]];
    return merge_symbols(v, ids, n, rk);
}

// Longest special token starting at s[i], if any (special strings are matched before the regex, tiktoken `encode`).
SMGX_HD bool special_at(const BpeView& v, const uint8_t* s, uint32_t i, uint32_t n, uint32_t& len, uint32_t& id) {
    const uint8_t c = s[i];
    if (!((v.special_first[c >> 5] >> (c & 31)) & 1)) return false;
    bool found = false;
    for (uint32_t k = 0; k < v.n_special; ++k) {
        const SpecialTok t = v.specials[k];
        if (t.len > n - i || (found && t.len <= len)) continue;
        bool eq = true;
        for (uint32_t b = 0; b < t.len; ++b) if (v.blob[t.off + b] != s[i + b]) { eq = false; break; }
        if (eq) { found = true; len = t.len; id = t.id; }
    }
    return found;
}

}  // namespace smgx
