// K1 — GPU tokenizer: vocabulary tables + pre-tokenise / BPE / compaction kernels.  See tokenizer.h and bpe.cuh.
#include "tokenizer.h"

#include <algorithm>
#include <cstring>
#include <fstream>
#include <sstream>
#include <unordered_map>

#include "deepseek_tables.h"
#include "nfc_tables.h"
#include "unicode_tables.h"

namespace smgx {

namespace {

constexpr uint32_t kInvalidTok = 0xFFFFFFFFu;

// Per-request kernels (the K1a candidates, pre-tokenizer, NFC and ▁ stages) run on a grid of request_grid(chunks, n): blockIdx.x = 256-byte
// chunk of the request, one thread per byte; the request index is folded over y and z because gridDim.y is capped at 65535, and
// request_index() unfolds it.  The last z slice can hold up to gridDim.z - 1 indices ≥ n: those CTAs return before reading offsets.
constexpr uint32_t kMaxGridY = 65535;
dim3 request_grid(uint32_t chunks, uint32_t n) {
    SMGX_REQUIRE(n >= 1 && (uint64_t)n <= (uint64_t)kMaxGridY * kMaxGridY, "request grid: batch size out of range");   // gridDim.z ≤ 65535 too
    const uint32_t z = (uint32_t)(((uint64_t)n + kMaxGridY - 1) / kMaxGridY);
    return dim3(chunks, (n + z - 1) / z, z);
}
__device__ __forceinline__ uint32_t request_index() { return blockIdx.z * gridDim.y + blockIdx.y; }

// ---- K1a: pre-tokenisation, parallel over bytes ---------------------------------------------------------------
// Special tokens first (tiktoken `encode`: the regex only ever sees the text between two specials):
//   special_candidates_kernel   does a special string start at this byte?  (longest at a position)
//   special_resolve_kernel      one warp per request: accept candidates left to right, dropping those inside an accepted span
//   flags: 0 ordinary byte, 1 piece start, 2 first byte of a special, 3 inside a special, 4 unresolved candidate
__global__ void __launch_bounds__(256) special_candidates_kernel(BpeView v, const uint8_t* __restrict__ text, const uint32_t* __restrict__ offsets,
                                                                 uint32_t n, uint8_t* __restrict__ flags, uint32_t* __restrict__ tmp_ids,
                                                                 uint64_t* __restrict__ tmp_rk) {
    const uint32_t r = request_index();
    if (r >= n) return;
    const uint32_t beg = offsets[r], rend = offsets[r + 1];
    const uint32_t i = beg + blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= rend) return;
    const uint8_t c = text[i];
    if (!((v.special_first[c >> 5] >> (c & 31)) & 1)) return;
    uint32_t len, id;
    if (special_at(v, text, i, rend, len, id)) { flags[i] = 4; tmp_ids[i] = id; tmp_rk[i] = len; }
}
__global__ void __launch_bounds__(256) special_resolve_kernel(const uint32_t* __restrict__ offsets, uint32_t n, uint8_t* __restrict__ flags,
                                                              uint32_t* __restrict__ tmp_ids, const uint64_t* __restrict__ tmp_rk,
                                                              uint32_t* __restrict__ totals) {
    const int lane = threadIdx.x & 31;
    const uint32_t r = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (r >= n) return;
    const uint32_t beg = offsets[r], end = offsets[r + 1];
    uint32_t skip_until = beg, count = 0;
    for (uint32_t base = beg; base < end; base += 32) {
        const uint32_t i = base + lane;
        unsigned m = __ballot_sync(0xffffffffu, i < end && flags[i] == 4);
        while (m) {
            const int k = __ffs((int)m) - 1;
            m &= m - 1;
            const uint32_t p = base + k;
            if (p < skip_until) { if (lane == 0) flags[p] = 0; continue; }   // starts inside an accepted special
            const uint32_t len = (uint32_t)tmp_rk[p];
            for (uint32_t j = lane; j < len; j += 32) {
                flags[p + j] = j == 0 ? 2 : 3;
                if (j) tmp_ids[p + j] = 0xFFFFFFFFu;
            }
            skip_until = p + len;
            ++count;
        }
        __syncwarp();
    }
    if (lane == 0) totals[r] = count;
}

// The regex scan itself.  Positions where a piece MUST start whatever came before — the end of a letter run (every
// alternative that consumes a letter stops at the end of the run or hands over to one that does), both ends of a digit
// run (digits are consumed by \p{N}{1,3} only), the start of the request and the byte after a special — cut the text
// into short independent segments; one thread per such "anchor" replays the hand-compiled regex until the next anchor
// and appends every piece it finds to a dense piece list (CTA-staged, one global atomic per CTA).  The r50k pattern has its
// own anchor rule (bpe.cuh: r50k_anchor_rule); the cl100k one is wrong there (" 123" is one r50k piece).
struct Piece { uint32_t start, len, req; };

__device__ __forceinline__ bool is_anchor(const uint8_t* s, uint32_t i, uint32_t beg, const uint8_t* flags, const UnicodeView& u) {
    if (i == beg) return true;
    if (flags[i - 1] >= 2) return true;                      // byte after a special token
    uint32_t l;
    const uint8_t c = char_class(utf8_decode(s, i, i + 4, l), u);   // valid UTF-8: a lead byte's continuation bytes exist
    const uint8_t pc = char_class(prev_cp(s, i, beg), u);
    return (pc == CH_LETTER && c != CH_LETTER) || (c == CH_NUMBER) != (pc == CH_NUMBER);
}
// Window form of next_piece_cl100k: the CTA's 256-byte window is classified ONCE into shared memory (phase 0 of the kernel:
// s_cls[k] = class | utf-8 length << 4 for a lead byte, kCont for a continuation byte; s_stop[k] = first byte of a special) and
// the regex then runs on classes instead of decoding and binary-searching every code point again.  Same alternatives, same order,
// same analytic resolution of the look-ahead as next_piece_cl100k; whenever a decision needs a byte beyond the window (and the
// window does not end the request) it returns kBail and the caller falls back to the global-memory matcher for that piece.
// kDigits as in next_piece_llama: 3 for cl100k, 1 for Qwen2.
constexpr uint8_t kCont = 0x0F;
constexpr uint32_t kBail = 0xFFFFFFFFu;
template <int kDigits>
__device__ __forceinline__ uint32_t next_piece_window(const uint8_t* __restrict__ s_txt, const uint8_t* __restrict__ s_cls, const uint8_t* __restrict__ s_stop,
                                                      uint32_t k, uint32_t W, bool ends_text) {
#define WIN_NEED(j) do { if ((j) >= W && !ends_text) return kBail; } while (0)
#define WIN_END(j) ((j) >= W || s_stop[(j)])
    const uint8_t c0 = s_cls[k] & 0x0F;
    const uint32_t len0 = s_cls[k] >> 4;
    const uint8_t b0 = s_txt[k];
    // 1. (?i:'s|'t|'re|'ve|'m|'ll|'d)  (+ U+017F for 's')
    if (b0 == '\'') {
        WIN_NEED(k + 1);
        if (!WIN_END(k + 1)) {
            const uint8_t b1 = s_txt[k + 1];
            if (b1 < 0x80) {
                const uint32_t c1 = b1 | 0x20;
                if (c1 == 's' || c1 == 't' || c1 == 'm' || c1 == 'd') return k + 2;
                WIN_NEED(k + 2);
                if (!WIN_END(k + 2) && s_txt[k + 2] < 0x80) {
                    const uint32_t c2 = s_txt[k + 2] | 0x20;
                    if ((c1 == 'r' && c2 == 'e') || (c1 == 'v' && c2 == 'e') || (c1 == 'l' && c2 == 'l')) return k + 3;
                }
            } else {
                WIN_NEED(k + 2);
                if (k + 2 < W && b1 == 0xC5 && s_txt[k + 2] == 0xBF) return k + 3;   // 'ſ
            }
        }
    }
    const bool nl0 = b0 == '\n' || b0 == '\r';
    // 2. [^\r\n\p{L}\p{N}]?\p{L}+
    {
        uint32_t j = k;
        bool ok = c0 == CH_LETTER;
        if (!ok && c0 != CH_NUMBER && !nl0) {
            const uint32_t k1 = k + len0;
            WIN_NEED(k1);
            if (!WIN_END(k1) && (s_cls[k1] & 0x0F) == CH_LETTER) { j = k1; ok = true; }
        }
        if (ok) {
            for (;;) {
                WIN_NEED(j);
                if (WIN_END(j) || (s_cls[j] & 0x0F) != CH_LETTER) break;
                j += s_cls[j] >> 4;
            }
            return j;
        }
    }
    // 3. \p{N}{1,3}  (Qwen2: \p{N})
    if (c0 == CH_NUMBER) {
        uint32_t j = k + len0;
        for (int c = 1; c < kDigits; ++c) {
            WIN_NEED(j);
            if (WIN_END(j) || (s_cls[j] & 0x0F) != CH_NUMBER) break;
            j += s_cls[j] >> 4;
        }
        return j;
    }
    // 4.  ?[^\s\p{L}\p{N}]+[\r\n]*
    {
        uint32_t j = k;
        bool ok = c0 == CH_OTHER;
        if (!ok && b0 == ' ') {
            WIN_NEED(k + 1);
            if (!WIN_END(k + 1) && (s_cls[k + 1] & 0x0F) == CH_OTHER) { j = k + 1; ok = true; }
        }
        if (ok) {
            for (;;) {
                WIN_NEED(j);
                if (WIN_END(j) || (s_cls[j] & 0x0F) != CH_OTHER) break;
                j += s_cls[j] >> 4;
            }
            for (;;) {
                WIN_NEED(j);
                if (WIN_END(j) || !(s_txt[j] == '\n' || s_txt[j] == '\r')) break;
                ++j;
            }
            return j;
        }
    }
    // 5-7. whitespace run starting at k
    uint32_t j = k, last_nl_end = 0, last_start = k, count = 0;
    for (;;) {
        WIN_NEED(j);
        if (WIN_END(j) || (s_cls[j] & 0x0F) != CH_SPACE) break;
        last_start = j;
        const bool nl = s_txt[j] == '\n' || s_txt[j] == '\r';
        j += s_cls[j] >> 4;
        ++count;
        if (nl) last_nl_end = j;
    }
    if (last_nl_end) return last_nl_end;   // 5. \s*[\r\n]+
    if (WIN_END(j)) return j;              // 6. \s+(?!\S): the run reaches the end of the (slice of) text
    if (count >= 2) return last_start;     // 6. give back one char so that whitespace follows
    return j;                              // 7. \s+
#undef WIN_NEED
#undef WIN_END
}

// Window form of next_piece_r50k, same contract as next_piece_window (kBail when a decision needs a byte beyond the window).
__device__ __forceinline__ uint32_t next_piece_window_r50k(const uint8_t* __restrict__ s_txt, const uint8_t* __restrict__ s_cls, const uint8_t* __restrict__ s_stop,
                                                           uint32_t k, uint32_t W, bool ends_text) {
#define WIN_NEED(j) do { if ((j) >= W && !ends_text) return kBail; } while (0)
#define WIN_END(j) ((j) >= W || s_stop[(j)])
    const uint8_t c0 = s_cls[k] & 0x0F;
    const uint8_t b0 = s_txt[k];
    // 1. 's|'t|'re|'ve|'m|'ll|'d  (case-sensitive)
    if (b0 == '\'') {
        WIN_NEED(k + 1);
        if (!WIN_END(k + 1)) {
            const uint8_t b1 = s_txt[k + 1];
            if (b1 == 's' || b1 == 't' || b1 == 'm' || b1 == 'd') return k + 2;
            if (b1 == 'r' || b1 == 'v' || b1 == 'l') {
                WIN_NEED(k + 2);
                if (!WIN_END(k + 2) && (b1 == 'l' ? s_txt[k + 2] == 'l' : s_txt[k + 2] == 'e')) return k + 3;
            }
        }
    }
    // 2-4.  ?\p{L}+ |  ?\p{N}+ |  ?[^\s\p{L}\p{N}]+  — a run of one non-space class, optionally led by one U+0020
    {
        uint32_t j = k;
        uint8_t rc = c0;
        if (b0 == ' ') {
            WIN_NEED(k + 1);
            if (!WIN_END(k + 1) && (s_cls[k + 1] & 0x0F) != CH_SPACE) { j = k + 1; rc = s_cls[k + 1] & 0x0F; }
        }
        if (rc != CH_SPACE) {
            for (;;) {
                WIN_NEED(j);
                if (WIN_END(j) || (s_cls[j] & 0x0F) != rc) break;
                j += s_cls[j] >> 4;
            }
            return j;
        }
    }
    // 5-6. whitespace run starting at k
    uint32_t j = k, last_start = k, count = 0;
    for (;;) {
        WIN_NEED(j);
        if (WIN_END(j) || (s_cls[j] & 0x0F) != CH_SPACE) break;
        last_start = j;
        j += s_cls[j] >> 4;
        ++count;
    }
    if (WIN_END(j)) return j;              // 5. \s+(?!\S): the run reaches the end of the (slice of) text
    if (count >= 2) return last_start;     // 5. give back one char so that whitespace follows
    return j;                              // 6. \s+
#undef WIN_NEED
#undef WIN_END
}

// Window form of next_piece_deepseek, same contract as next_piece_window.  s_cls holds ds_class() (kana flag included) | length << 4.
__device__ __forceinline__ uint32_t next_piece_window_deepseek(const uint8_t* __restrict__ s_txt, const uint8_t* __restrict__ s_cls,
                                                               const uint8_t* __restrict__ s_stop, uint32_t k, uint32_t W, bool ends_text) {
#define WIN_NEED(j) do { if ((j) >= W && !ends_text) return kBail; } while (0)
#define WIN_END(j) ((j) >= W || s_stop[(j)])
#define WIN_AT(j) (WIN_END(j) ? kDsEnd : ds_stage_class(s_cls[(j)] & 0x0F, z))
    const uint8_t c0 = s_cls[k] & 0x0F;
    const uint32_t len0 = s_cls[k] >> 4;
    const uint8_t b0 = s_txt[k];
    // Split 1: \p{N}{1,3}
    if (c0 == DS_N) {
        uint32_t j = k + len0;
        for (int c = 1; c < 3; ++c) {
            WIN_NEED(j);
            if (WIN_END(j) || (s_cls[j] & 0x0F) != DS_N) break;
            j += s_cls[j] >> 4;
        }
        return j;
    }
    // Split 3 inside the stage piece of zone z
    const uint8_t z = c0 & DS_KANA, c = c0 & 7;
    // 1. [ASCII punctuation][A-Za-z]+
    if (b0 < 0x80 && ds_punct_or_symbol(c)) {
        uint32_t j = k + 1;
        for (;;) {
            WIN_NEED(j);
            if (WIN_END(j) || !is_ascii_letter(s_txt[j])) break;
            ++j;
        }
        if (j > k + 1) return j;
    }
    // 2. [^\r\n\p{L}\p{P}\p{S}]?[\p{L}\p{M}]+
    {
        uint32_t j = k;
        bool ok = ds_letter_or_mark(c);
        if (!ok && !ds_punct_or_symbol(c) && b0 != '\n' && b0 != '\r') {
            WIN_NEED(k + len0);
            if (ds_letter_or_mark(WIN_AT(k + len0))) { j = k + len0; ok = true; }
        }
        if (ok) {
            for (;;) {
                WIN_NEED(j);
                if (!ds_letter_or_mark(WIN_AT(j))) break;
                j += s_cls[j] >> 4;
            }
            return j;
        }
    }
    // 3.  ?[\p{P}\p{S}]+[\r\n]*
    {
        uint32_t j = k;
        bool ok = ds_punct_or_symbol(c);
        if (!ok && b0 == ' ') {
            WIN_NEED(k + 1);
            if (ds_punct_or_symbol(WIN_AT(k + 1))) { j = k + 1; ok = true; }
        }
        if (ok) {
            for (;;) {
                WIN_NEED(j);
                if (!ds_punct_or_symbol(WIN_AT(j))) break;
                j += s_cls[j] >> 4;
            }
            for (;;) {
                WIN_NEED(j);
                if (WIN_AT(j) != DS_WS || !(s_txt[j] == '\n' || s_txt[j] == '\r')) break;
                ++j;
            }
            return j;
        }
    }
    // 4-6. whitespace run starting at k
    if (c == DS_WS) {
        uint32_t j = k, last_nl_end = 0;
        for (;;) {
            WIN_NEED(j);
            if (WIN_AT(j) != DS_WS) break;
            const bool nl = s_txt[j] == '\n' || s_txt[j] == '\r';
            j += s_cls[j] >> 4;
            if (nl) last_nl_end = j;
        }
        if (last_nl_end) return last_nl_end;   // 4. \s*[\r\n]+
        if (WIN_AT(j) == kDsEnd) return j;     // 5. \s+(?!\S): the run reaches the end of the stage piece
        if (j == k + len0) return j;           // 6. \s+: a single whitespace character
        do --j; while (s_cls[j] == kCont);     // 5. give back the last character so that whitespace follows
        return j;
    }
    // a gap: "other" characters up to the first where an alternative matches
    uint32_t j = k + len0;
    for (;;) {
        WIN_NEED(j);
        if (WIN_AT(j) != DS_OTHER) break;
        const uint32_t j1 = j + (s_cls[j] >> 4);
        WIN_NEED(j1);
        if (ds_letter_or_mark(WIN_AT(j1))) break;
        j = j1;
    }
    return j;
#undef WIN_NEED
#undef WIN_END
#undef WIN_AT
}

// The global-memory DeepSeek matcher runs only for pieces that cross a window; as a call rather than inlined into the replay loop it keeps
// the kernel from spilling (inlined, ptxas holds the kernel at 32 registers and spills the replay loop's state).
__device__ __noinline__ uint32_t next_piece_deepseek_global(const uint8_t* s, uint32_t i, uint32_t n, UnicodeView u, const uint8_t* stop) {
    return next_piece_deepseek(s, i, n, u, stop);
}

// One kernel per pattern: the instantiations share the window classification, anchor packing and piece flush, and differ in the anchor
// rule and the two matchers.
template <Pretok P>
__global__ void __launch_bounds__(256) pretokenize_kernel(BpeView v, const uint8_t* __restrict__ text, const uint32_t* __restrict__ offsets,
                                                          uint32_t n, uint8_t* __restrict__ flags, Piece* __restrict__ pieces,
                                                          uint32_t* __restrict__ n_pieces) {
    __shared__ Piece s_list[320];
    __shared__ uint32_t s_anchor[256];
    __shared__ uint32_t s_wcnt[8];
    __shared__ uint32_t s_count, s_base;
    __shared__ uint8_t s_txt[256], s_cls[256], s_stop[256], s_flag[256];
    const uint32_t r = request_index();
    if (r >= n) return;
    if (threadIdx.x == 0) s_count = 0;
    const uint32_t beg = offsets[r], rend = offsets[r + 1];
    const uint32_t cstart = beg + blockIdx.x * blockDim.x;
    const uint32_t i = cstart + threadIdx.x;
    const uint32_t W = cstart < rend ? min(256u, rend - cstart) : 0;
    const bool ends_text = cstart + W == rend;
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    // phase 0 (every thread, one byte each): classify the window once
    if (threadIdx.x < W) {
        const uint8_t b = text[i], fl = flags[i];
        s_txt[threadIdx.x] = b;
        s_flag[threadIdx.x] = fl;
        s_stop[threadIdx.x] = fl == 2;
        if ((b & 0xC0) == 0x80) s_cls[threadIdx.x] = kCont;
        else if constexpr (P == Pretok::DeepSeek) {   // v.uni holds the deepseek_tables.h ranges
            uint32_t l; const uint32_t cp = utf8_decode(text, i, rend, l); s_cls[threadIdx.x] = (uint8_t)(ds_class(cp, v.uni) | (l << 4));
        }
        else { uint32_t l; const uint32_t cp = utf8_decode(text, i, rend, l); s_cls[threadIdx.x] = (uint8_t)(char_class(cp, v.uni) | (l << 4)); }
    }
    __syncthreads();
    // anchor test on the window (is_anchor on classes); the char before the window is classified from global memory
    auto anchor_at = [&](uint32_t k) -> bool {   // k < W, lead byte, not inside a special
        const uint32_t gi = cstart + k;
        if (gi == beg) return true;
        if ((k ? s_flag[k - 1] : flags[gi - 1]) >= 2) return true;
        const uint8_t c = s_cls[k] & 0x0F;
        uint8_t pc;
        int q = (int)k - 1;
        while (q >= 0 && s_cls[q] == kCont) --q;
        if (q >= 0) pc = s_cls[q] & 0x0F;
        else if constexpr (P == Pretok::DeepSeek) pc = ds_class(prev_cp(text, gi, beg), v.uni);
        else pc = char_class(prev_cp(text, gi, beg), v.uni);
        if constexpr (P == Pretok::R50k) return r50k_anchor_rule(pc, k ? s_txt[k - 1] : text[gi - 1], c, s_txt[k]);
        else if constexpr (P == Pretok::Qwen2) return qwen2_anchor_rule(pc, c);
        else if constexpr (P == Pretok::DeepSeek) return deepseek_anchor_rule(pc, c);
        else return (pc == CH_LETTER && c != CH_LETTER) || (c == CH_NUMBER) != (pc == CH_NUMBER);
    };
    // phase 1: which bytes are anchors?  They are then packed densely, so that phase 2 — the serial regex replay — runs with full
    // warps instead of one live lane in six.
    const bool anchor = threadIdx.x < W && s_cls[threadIdx.x] != kCont && s_flag[threadIdx.x] < 2 && anchor_at(threadIdx.x);
    const unsigned bal = __ballot_sync(0xffffffffu, anchor);
    if (lane == 0) s_wcnt[wid] = (uint32_t)__popc(bal);
    __syncthreads();
    uint32_t before = 0, n_anchor = 0;
#pragma unroll
    for (int w = 0; w < 8; ++w) { const uint32_t c = s_wcnt[w]; if (w < wid) before += c; n_anchor += c; }
    if (anchor) s_anchor[before + (uint32_t)__popc(bal & ((1u << lane) - 1u))] = threadIdx.x;
    __syncthreads();
    // phase 2: thread k replays the regex from the k-th anchor up to the next one; a special's first byte (flags == 2) ends the
    // slice.  The warp iterates in lockstep (one piece per live lane and round).
    if ((uint32_t)(wid * 32) < n_anchor) {
        bool live = threadIdx.x < n_anchor;
        uint32_t p = live ? cstart + s_anchor[threadIdx.x] : 0;
        while (__any_sync(0xffffffffu, live)) {
            if (live) {
                flags[p] = 1;
                uint32_t q = kBail;
                if (p - cstart < W) {
                    uint32_t e;
                    if constexpr (P == Pretok::R50k) e = next_piece_window_r50k(s_txt, s_cls, s_stop, p - cstart, W, ends_text);
                    else if constexpr (P == Pretok::Qwen2) e = next_piece_window<1>(s_txt, s_cls, s_stop, p - cstart, W, ends_text);
                    else if constexpr (P == Pretok::DeepSeek) e = next_piece_window_deepseek(s_txt, s_cls, s_stop, p - cstart, W, ends_text);
                    else e = next_piece_window<3>(s_txt, s_cls, s_stop, p - cstart, W, ends_text);
                    if (e != kBail) q = cstart + e;
                }
                if (q == kBail) {   // the piece looks beyond the window
                    if constexpr (P == Pretok::R50k) q = next_piece_r50k(text, p, rend, v.uni, flags);
                    else if constexpr (P == Pretok::Qwen2) q = next_piece_qwen2(text, p, rend, v.uni, flags);
                    else if constexpr (P == Pretok::DeepSeek) q = next_piece_deepseek_global(text, p, rend, v.uni, flags);
                    else q = next_piece_cl100k(text, p, rend, v.uni, flags);
                }
                const uint32_t slot = atomicAdd(&s_count, 1u);
                if (slot < 320) s_list[slot] = Piece{p, q - p, r};
                else { const uint32_t g = atomicAdd(n_pieces, 1u); pieces[g] = Piece{p, q - p, r}; }   // overflow: straight to the global list
                bool stop;
                if (q >= rend) stop = true;
                else if (q - cstart < W) stop = s_flag[q - cstart] == 2 || anchor_at(q - cstart);
                else if constexpr (P == Pretok::R50k) stop = flags[q] == 2 || is_anchor_r50k(text, q, beg, flags, v.uni);
                else if constexpr (P == Pretok::Qwen2) stop = flags[q] == 2 || is_anchor_qwen2(text, q, beg, flags, v.uni);
                else if constexpr (P == Pretok::DeepSeek) stop = flags[q] == 2 || is_anchor_deepseek(text, q, beg, flags, v.uni);
                else stop = flags[q] == 2 || is_anchor(text, q, beg, flags, v.uni);
                if (stop) live = false; else p = q;
            }
        }
    }
    __syncthreads();
    const uint32_t cnt = s_count < 320 ? s_count : 320;
    if (threadIdx.x == 0 && cnt) s_base = atomicAdd(n_pieces, cnt);
    __syncthreads();
    for (uint32_t k = threadIdx.x; k < cnt; k += blockDim.x) pieces[s_base + k] = s_list[k];
}

// K1b: BPE over the dense piece list, three kernels so that every one of them runs on full warps:
//   bpe_lookup_kernel   thread per piece: whole-piece vocabulary hit → one token (most pieces of natural text); misses are appended to
//                       two lists — pieces of ≤ kSmemSyms bytes and longer ones (warp-aggregated atomics)
//   bpe_merge_kernel    thread per short miss: tiktoken's byte-pair merge with symbols and pair ranks in shared memory (column per
//                       thread); the warp runs the merge loop in lockstep, one merge per live lane and round
//   bpe_long_kernel     warp per long miss (indentation runs, rules of dashes, URLs …): up to 32 bytes one symbol per lane, the
//                       leftmost-lowest-rank pair found with one redux.sync per merge, the tail shifted down by shuffles; up to 256
//                       bytes a linked list in shared memory with a strided minimum scan; beyond that (very rare) lane 0 merges in
//                       place in the global scratch
// Unused slots of a piece are set INVALID for the compaction.  counters: [0] pieces, [1] short misses, [2] long misses.
constexpr uint32_t kSmemSyms = 15;
constexpr uint32_t kLongSyms = 256;   // longest piece the warp-per-piece kernel keeps in shared memory
__global__ void __launch_bounds__(256) bpe_lookup_kernel(BpeView v, const uint8_t* __restrict__ text, const Piece* __restrict__ pieces,
                                                         uint32_t* __restrict__ counters, uint32_t* __restrict__ tmp_ids, uint32_t* __restrict__ totals,
                                                         uint32_t* __restrict__ miss_short, uint32_t* __restrict__ miss_long) {
    const uint32_t np = counters[0];
    const int lane = threadIdx.x & 31;
    const uint32_t stride = gridDim.x * blockDim.x;
    for (uint32_t t0 = blockIdx.x * blockDim.x; t0 < np; t0 += stride) {
        const uint32_t t = t0 + threadIdx.x;
        int kind = 0;   // 1 short miss, 2 long miss
        if (t < np) {
            const Piece pc = pieces[t];
            uint32_t id;
            if (v.whole_piece && piece_lookup(v, text + pc.start, pc.len, id)) {
                tmp_ids[pc.start] = id;
                for (uint32_t j = pc.start + 1; j < pc.start + pc.len; ++j) tmp_ids[j] = kInvalidTok;
                atomicAdd(&totals[pc.req], 1u);
            } else kind = pc.len <= kSmemSyms ? 1 : 2;
        }
#pragma unroll
        for (int k = 1; k <= 2; ++k) {
            const unsigned bal = __ballot_sync(0xffffffffu, kind == k);
            if (!bal) continue;
            uint32_t base = 0;
            if (lane == __ffs((int)bal) - 1) base = atomicAdd(&counters[k], (uint32_t)__popc(bal));
            base = __shfl_sync(0xffffffffu, base, __ffs((int)bal) - 1);
            if (kind == k) (k == 1 ? miss_short : miss_long)[base + (uint32_t)__popc(bal & ((1u << lane) - 1u))] = t;
        }
    }
}

// kChar (SentencePiece-style BPE): the initial symbols are not the piece's bytes but what ms_symbolize_kernel left in the piece's slots of
// tmp_ids (code-point ids and byte-fallback tokens, kInvalidTok between them), and the tiers go by symbol count, not byte length.
template <bool kChar>
__global__ void __launch_bounds__(256) bpe_merge_kernel(BpeView v, const uint8_t* __restrict__ text, const Piece* __restrict__ pieces,
                                                        const uint32_t* __restrict__ counters, const uint32_t* __restrict__ miss_short,
                                                        uint32_t* __restrict__ tmp_ids, uint32_t* __restrict__ totals) {
    __shared__ uint32_t s_id[kSmemSyms][256];     // symbol ids
    __shared__ uint32_t s_rank[kSmemSyms][256];   // rank of the pair (i, i+1); kRankMax = no merge
    __shared__ uint32_t s_mid[kSmemSyms][256];    // id that pair merges into
    const uint32_t n = counters[1], tid = threadIdx.x;
    const uint32_t stride = gridDim.x * blockDim.x;
    for (uint32_t t0 = blockIdx.x * blockDim.x; t0 < n; t0 += stride) {   // t0 is CTA-uniform: whole warps stay in the loop together
        const bool valid = t0 + tid < n;
        Piece pc{0, 0, 0};
        if (valid) pc = pieces[miss_short[t0 + tid]];
        const uint32_t i = pc.start, plen = pc.len;
        uint32_t m = plen;
        if (valid) {
            if constexpr (kChar) {
                m = 0;
                for (uint32_t j = 0; j < plen; ++j) { const uint32_t id = tmp_ids[i + j]; if (id != kInvalidTok) s_id[m++][tid] = id; }
            } else {
                for (uint32_t j = 0; j < plen; ++j) s_id[j][tid] = v.byte_token[text[i + j]];
            }
            for (uint32_t j = 0; j + 1 < m; ++j) {
                const uint64_t pr = pair_lookup(v, s_id[j][tid], s_id[j + 1][tid]);
                s_rank[j][tid] = (uint32_t)(pr >> 32); s_mid[j][tid] = (uint32_t)pr;
            }
        }
        bool merging = valid && m >= 2;
        while (__any_sync(0xffffffffu, merging)) {
            if (merging) {
                uint32_t best = kRankMax, bi = 0;
                for (uint32_t j = 0; j + 1 < m; ++j) { const uint32_t rk = s_rank[j][tid]; if (rk < best) { best = rk; bi = j; } }   // leftmost minimum
                if (best == kRankMax) merging = false;
                else {
                    s_id[bi][tid] = s_mid[bi][tid];
                    for (uint32_t j = bi + 1; j + 1 < m; ++j) { s_id[j][tid] = s_id[j + 1][tid]; s_rank[j][tid] = s_rank[j + 1][tid]; s_mid[j][tid] = s_mid[j + 1][tid]; }
                    --m;
                    if (bi + 1 < m) { const uint64_t pr = pair_lookup(v, s_id[bi][tid], s_id[bi + 1][tid]); s_rank[bi][tid] = (uint32_t)(pr >> 32); s_mid[bi][tid] = (uint32_t)pr; }
                    else s_rank[bi][tid] = kRankMax;
                    if (bi > 0) { const uint64_t pr = pair_lookup(v, s_id[bi - 1][tid], s_id[bi][tid]); s_rank[bi - 1][tid] = (uint32_t)(pr >> 32); s_mid[bi - 1][tid] = (uint32_t)pr; }
                    if (m < 2) merging = false;
                }
            }
        }
        if (valid) {
            for (uint32_t j = 0; j < m; ++j) tmp_ids[i + j] = s_id[j][tid];
            for (uint32_t j = i + m; j < i + plen; ++j) tmp_ids[j] = kInvalidTok;
            atomicAdd(&totals[pc.req], m);
        }
    }
}

// kChar: pack the symbols of a piece's slots tmp_ids[i .. i+plen) (kInvalidTok between them) into w[0 ..); w may be those slots themselves
// (a lane writes at or below the index it read, and every read of a round precedes its writes).
__device__ __forceinline__ void gather_symbols(const uint32_t* tmp_ids, uint32_t i, uint32_t plen, uint32_t* w, int lane) {
    uint32_t written = 0;
    for (uint32_t base = 0; base < plen; base += 32) {
        const uint32_t j = base + lane;
        const uint32_t id = j < plen ? tmp_ids[i + j] : kInvalidTok;
        const unsigned bal = __ballot_sync(0xffffffffu, id != kInvalidTok);
        if (id != kInvalidTok) w[written + (uint32_t)__popc(bal & ((1u << lane) - 1u))] = id;
        written += (uint32_t)__popc(bal);
    }
    __syncwarp();
}

template <bool kChar>
__global__ void __launch_bounds__(256) bpe_long_kernel(BpeView v, const uint8_t* __restrict__ text, const Piece* __restrict__ pieces,
                                                       const uint32_t* __restrict__ counters, const uint32_t* __restrict__ miss_long,
                                                       uint32_t* __restrict__ tmp_ids, uint64_t* __restrict__ tmp_rk, uint32_t* __restrict__ totals) {
    __shared__ uint32_t s_id[8][kLongSyms], s_rank[8][kLongSyms], s_mid[8][kLongSyms];
    __shared__ uint16_t s_nxt[8][kLongSyms], s_prv[8][kLongSyms];
    const uint32_t n = counters[2];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const uint32_t nw = gridDim.x * (blockDim.x >> 5);
    for (uint32_t k = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; k < n; k += nw) {
        const Piece pc = pieces[miss_long[k]];
        const uint32_t i = pc.start, plen = pc.len;
        uint32_t ns = plen;   // initial symbols
        if constexpr (kChar) {
            ns = 0;
            for (uint32_t base = 0; base < plen; base += 32)
                ns += (uint32_t)__popc(__ballot_sync(0xffffffffu, base + lane < plen && tmp_ids[i + base + lane] != kInvalidTok));
        }
        uint32_t m;
        if (ns <= 32) {
            m = ns;
            uint32_t id;
            if constexpr (kChar) {
                gather_symbols(tmp_ids, i, plen, s_id[wid], lane);
                id = (uint32_t)lane < ns ? s_id[wid][lane] : 0;
                __syncwarp();
            } else {
                id = (uint32_t)lane < plen ? v.byte_token[text[i + lane]] : 0;
            }
            uint32_t nid = __shfl_down_sync(0xffffffffu, id, 1);
            uint32_t rank = kRankMax, mid = 0;
            if ((uint32_t)lane + 1 < m) { const uint64_t pr = pair_lookup(v, id, nid); rank = (uint32_t)(pr >> 32); mid = (uint32_t)pr; }
            for (;;) {
                // ranks are vocabulary positions (< 2^27), so rank * 32 + lane orders by rank, then by position
                const uint32_t key = ((uint32_t)lane + 1 < m && rank != kRankMax) ? ((rank << 5) | (uint32_t)lane) : 0xFFFFFFFFu;
                const uint32_t kmin = __reduce_min_sync(0xffffffffu, key);
                if (kmin == 0xFFFFFFFFu) break;
                const int bi = (int)(kmin & 31u);
                if (lane == bi) id = mid;
                const uint32_t id_dn = __shfl_down_sync(0xffffffffu, id, 1), rank_dn = __shfl_down_sync(0xffffffffu, rank, 1), mid_dn = __shfl_down_sync(0xffffffffu, mid, 1);
                if (lane > bi) { id = id_dn; rank = rank_dn; mid = mid_dn; }
                --m;
                nid = __shfl_down_sync(0xffffffffu, id, 1);
                if (lane == bi || lane == bi - 1) {
                    rank = kRankMax;
                    if ((uint32_t)lane + 1 < m) { const uint64_t pr = pair_lookup(v, id, nid); rank = (uint32_t)(pr >> 32); mid = (uint32_t)pr; }
                }
            }
            if constexpr (kChar) {
                if ((uint32_t)lane < m) tmp_ids[i + lane] = id;
                for (uint32_t j = m + lane; j < plen; j += 32) tmp_ids[i + j] = kInvalidTok;
            } else {
                if ((uint32_t)lane < plen) tmp_ids[i + lane] = (uint32_t)lane < m ? id : kInvalidTok;
            }
        } else if (ns <= kLongSyms) {
            // 33 … kLongSyms symbols: symbols stay in place in shared memory, linked by next/prev indices (list order = index order, so
            // "leftmost" = smallest index); a merge unlinks one symbol and re-ranks two pairs; the minimum is a strided scan + 2 redux
            uint32_t* w_id = s_id[wid]; uint32_t* w_rank = s_rank[wid]; uint32_t* w_mid = s_mid[wid];
            uint16_t* w_nxt = s_nxt[wid]; uint16_t* w_prv = s_prv[wid];
            if constexpr (kChar) gather_symbols(tmp_ids, i, plen, w_id, lane);
            for (uint32_t j = lane; j < ns; j += 32) {
                if constexpr (!kChar) w_id[j] = v.byte_token[text[i + j]];
                w_nxt[j] = (uint16_t)(j + 1); w_prv[j] = (uint16_t)(j ? j - 1 : 0xFFFF);
            }
            __syncwarp();
            for (uint32_t j = lane; j < ns; j += 32) {
                uint32_t rk = kRankMax, md = 0;
                if (j + 1 < ns) { const uint64_t pr = pair_lookup(v, w_id[j], w_id[j + 1]); rk = (uint32_t)(pr >> 32); md = (uint32_t)pr; }
                w_rank[j] = rk; w_mid[j] = md;
            }
            __syncwarp();
            m = ns;
            for (;;) {
                uint32_t best = kRankMax, bpos = 0xFFFFFFFFu;
                for (uint32_t j = lane; j < ns; j += 32) { const uint32_t rk = w_rank[j]; if (rk < best) { best = rk; bpos = j; } }   // ascending j: leftmost per lane
                const uint32_t rmin = __reduce_min_sync(0xffffffffu, best);
                if (rmin == kRankMax) break;
                const uint32_t b = __reduce_min_sync(0xffffffffu, best == rmin ? bpos : 0xFFFFFFFFu);
                const uint32_t c = w_nxt[b], d = w_nxt[c], a = w_prv[b];
                __syncwarp();
                if (lane == 0) {
                    w_id[b] = w_mid[b]; w_nxt[b] = (uint16_t)d; w_rank[c] = kRankMax; w_id[c] = kInvalidTok;
                    if (d < ns) w_prv[d] = (uint16_t)b;
                }
                __syncwarp();
                if (lane == 0) {
                    uint32_t rk = kRankMax, md = 0;
                    if (d < ns) { const uint64_t pr = pair_lookup(v, w_id[b], w_id[d]); rk = (uint32_t)(pr >> 32); md = (uint32_t)pr; }
                    w_rank[b] = rk; w_mid[b] = md;
                } else if (lane == 1 && a != 0xFFFF) {
                    const uint64_t pr = pair_lookup(v, w_id[a], w_id[b]);
                    w_rank[a] = (uint32_t)(pr >> 32); w_mid[a] = (uint32_t)pr;
                }
                --m;
                __syncwarp();
            }
            uint32_t written = 0;   // compact the surviving symbols to the front of the piece's slots
            for (uint32_t base = 0; base < ns; base += 32) {
                const uint32_t j = base + lane;
                const bool alive = j < ns && w_id[j] != kInvalidTok;
                const unsigned bal = __ballot_sync(0xffffffffu, alive);
                if (alive) tmp_ids[i + written + (uint32_t)__popc(bal & ((1u << lane) - 1u))] = w_id[j];
                written += (uint32_t)__popc(bal);
            }
            for (uint32_t j = written + lane; j < plen; j += 32) tmp_ids[i + j] = kInvalidTok;
            __syncwarp();
        } else {
            m = 0;
            if constexpr (kChar) gather_symbols(tmp_ids, i, plen, tmp_ids + i, lane);   // in place
            if (lane == 0) {
                if constexpr (kChar) m = merge_symbols(v, tmp_ids + i, ns, tmp_rk + i);
                else m = byte_pair_merge(v, text + i, plen, tmp_ids + i, tmp_rk + i);
                for (uint32_t j = i + m; j < i + plen; ++j) tmp_ids[j] = kInvalidTok;
            }
            m = __shfl_sync(0xffffffffu, m, 0);
        }
        if (lane == 0) atomicAdd(&totals[pc.req], m);
    }
}

// exclusive scan of per-request token counts → token offsets (n + 1); one CTA, n ≤ a few 10^5
__global__ void __launch_bounds__(1024) scan_counts_kernel(const uint32_t* __restrict__ totals, uint32_t n, uint32_t* __restrict__ tok_offsets) {
    __shared__ uint32_t s_part[1024];
    __shared__ uint32_t s_carry;
    if (threadIdx.x == 0) s_carry = 0;
    __syncthreads();
    for (uint32_t base = 0; base < n; base += 1024) {
        uint32_t i = base + threadIdx.x;
        uint32_t x = i < n ? totals[i] : 0;
        s_part[threadIdx.x] = x;
        __syncthreads();
        for (uint32_t d = 1; d < 1024; d <<= 1) {
            uint32_t t = threadIdx.x >= d ? s_part[threadIdx.x - d] : 0;
            __syncthreads();
            s_part[threadIdx.x] += t;
            __syncthreads();
        }
        if (i < n) tok_offsets[i] = s_carry + s_part[threadIdx.x] - x;
        __syncthreads();
        if (threadIdx.x == 1023) s_carry += s_part[1023];
        __syncthreads();
    }
    if (threadIdx.x == 0) tok_offsets[n] = s_carry;
}

// K1c: one warp per request: stream-compact the valid token slots of its byte range into the ragged output
__global__ void __launch_bounds__(256) compact_tokens_kernel(const uint32_t* __restrict__ offsets, uint32_t n, const uint32_t* __restrict__ tmp_ids,
                                                             const uint32_t* __restrict__ tok_offsets, uint32_t* __restrict__ out_tokens) {
    const int lane = threadIdx.x & 31;
    const uint32_t r = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (r >= n) return;
    const uint32_t beg = offsets[r], end = offsets[r + 1];
    uint32_t out = tok_offsets[r];
    for (uint32_t base = beg; base < end; base += 32) {
        uint32_t i = base + lane;
        uint32_t v = i < end ? tmp_ids[i] : kInvalidTok;
        unsigned m = __ballot_sync(0xffffffffu, v != kInvalidTok);
        if (v != kInvalidTok) out_tokens[out + __popc(m & ((1u << lane) - 1u))] = v;
        out += __popc(m);
    }
}

// K1n: NFC normalization stage, only for a tokenizer loaded with a normalizer.  It runs after the specials are resolved on the RAW text
// (added tokens with normalized = false) and before the pre-tokenizer, and writes a normalized ragged copy of the batch — text, flags
// (2/3 of the specials carried over) and the specials' ids — that the pre-tokenizer, BPE and compaction then run on unchanged.
// Grids are sized for the raw text; nothing comes back to the host (the normalized length stays on the device).
//   nfc_check_kernel    thread per byte: does the request hold a code point that is not NFC-stable?  Most text does not (a clean
//                       request is its own NFC and is copied as it is)
//   nfc_segment_kernel  dirty requests, thread per byte: a segment starts at every NFC-stable code point, at the request start and
//                       after a special; its thread normalizes it in a 32-entry buffer into norm_tmp (3 bytes per input byte),
//                       or hands it to the long list; seg_len / chunk_sum / nlen collect the output lengths
//   nfc_long_kernel     warp per long segment (thousands of marks are legal): lane 0 normalizes it in global scratch, canonical
//                       ordering by a counting sort with the histogram in shared memory
//   scan_counts_kernel  normalized request lengths → offsets of the normalized batch
//   nfc_write_kernel    thread per byte: clean requests copy, dirty ones place every segment at (earlier chunks of the request +
//                       exclusive scan within the chunk)
constexpr uint32_t kNfcShort = 32;
struct NfcLong { uint32_t start, end, req; };

__global__ void __launch_bounds__(256) nfc_check_kernel(NfcView nv, const uint8_t* __restrict__ text, const uint32_t* __restrict__ offsets,
                                                        uint32_t n, const uint8_t* __restrict__ flags, uint32_t* __restrict__ dirty) {
    const uint32_t r = request_index();
    if (r >= n) return;
    const uint32_t beg = offsets[r], rend = offsets[r + 1];
    const uint32_t i = beg + blockIdx.x * blockDim.x + threadIdx.x;
    if (beg + blockIdx.x * blockDim.x >= rend) return;   // CTA-uniform
    bool bad = false;
    if (i < rend && text[i] >= 0xCC && flags[i] < 2) {   // lead byte of a code point ≥ U+0300 (everything below is stable)
        uint32_t l;
        bad = !nfc_stable(nv, utf8_decode(text, i, rend, l));
    }
    if (__any_sync(0xffffffffu, bad) && (threadIdx.x & 31) == 0) dirty[r] = 1;
}

__device__ __forceinline__ uint32_t block_sum_256(uint32_t x, uint32_t* s_w) {
    x = __reduce_add_sync(0xffffffffu, x);
    if ((threadIdx.x & 31) == 0) s_w[threadIdx.x >> 5] = x;
    __syncthreads();
    uint32_t t = 0;
#pragma unroll
    for (int w = 0; w < 8; ++w) t += s_w[w];
    __syncthreads();
    return t;
}

__global__ void __launch_bounds__(256) nfc_segment_kernel(NfcView nv, const uint8_t* __restrict__ text, const uint32_t* __restrict__ offsets,
                                                          uint32_t n, uint32_t first_byte, const uint8_t* __restrict__ flags,
                                                          const uint32_t* __restrict__ dirty, uint32_t* __restrict__ seg_len,
                                                          uint32_t* __restrict__ chunk_sum, uint32_t* __restrict__ nlen, uint8_t* __restrict__ norm_tmp,
                                                          NfcLong* __restrict__ longs, uint32_t* __restrict__ n_long) {
    __shared__ uint32_t s_w[8];
    const uint32_t r = request_index();
    if (r >= n) return;
    const uint32_t beg = offsets[r], rend = offsets[r + 1];
    const uint32_t cstart = beg + blockIdx.x * blockDim.x;
    if (cstart >= rend) return;
    if (!dirty[r]) {
        if (blockIdx.x == 0 && threadIdx.x == 0) nlen[r] = rend - beg;
        return;
    }
    const uint32_t i = cstart + threadIdx.x;
    uint32_t len = 0;
    if (i < rend) {
        const uint8_t fl = flags[i];
        if (fl >= 2) len = 1;   // special-token byte: copied as it is
        else if ((text[i] & 0xC0) != 0x80) {
            uint32_t l;
            const uint32_t cp = utf8_decode(text, i, rend, l);
            const bool stable = nfc_stable(nv, cp);
            if (stable || i == beg || flags[i - 1] >= 2) {
                const uint32_t e = nfc_segment_end(nv, text, i, rend, flags);
                uint8_t* out = norm_tmp + 3ull * (i - first_byte);
                if (stable && e == i + l) {   // a stable code point alone is its own NFC
                    for (uint32_t j = 0; j < l; ++j) out[j] = text[i + j];
                    len = l;
                } else {
                    uint32_t ent[kNfcShort];
                    uint32_t m = nfc_decompose_text(nv, text, i, e, ent, kNfcShort);
                    if (m <= kNfcShort) {
                        m = nfc_reorder_compose(nv, ent, m, nullptr, nullptr);
                        len = nfc_encode(ent, m, out);
                    } else {
                        longs[atomicAdd(n_long, 1u)] = NfcLong{i, e, r};
                    }
                }
            }
        }
        seg_len[i - first_byte] = len;
    }
    const uint32_t sum = block_sum_256(len, s_w);
    if (threadIdx.x == 0) {
        chunk_sum[cstart - first_byte] = sum;
        if (sum) atomicAdd(&nlen[r], sum);
    }
}

__global__ void __launch_bounds__(256) nfc_long_kernel(NfcView nv, const uint8_t* __restrict__ text, const uint32_t* __restrict__ offsets,
                                                       uint32_t first_byte, const NfcLong* __restrict__ longs, const uint32_t* __restrict__ n_long,
                                                       uint32_t* __restrict__ ent, uint32_t* __restrict__ seg_len, uint32_t* __restrict__ chunk_sum,
                                                       uint32_t* __restrict__ nlen, uint8_t* __restrict__ norm_tmp) {
    __shared__ uint32_t s_hist[8][256];
    const uint32_t n = *n_long;
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const uint32_t nw = gridDim.x * (blockDim.x >> 5);
    for (uint32_t k = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; k < n; k += nw) {
        if (lane != 0) continue;
        const NfcLong sg = longs[k];
        const uint64_t rel = sg.start - first_byte;
        const uint32_t cap = 2 * (sg.end - sg.start);   // at most two code points per byte (the generator asserts it)
        uint32_t* e = ent + 4 * rel;                     // [0, cap) the entries, [cap, 2 cap) the counting sort's buffer
        uint32_t m = nfc_decompose_text(nv, text, sg.start, sg.end, e, cap);
        m = nfc_reorder_compose(nv, e, m, e + cap, s_hist[wid]);
        const uint32_t len = nfc_encode(e, m, norm_tmp + 3 * rel);
        seg_len[rel] = len;
        const uint32_t beg = offsets[sg.req];
        atomicAdd(&chunk_sum[beg + (sg.start - beg) / 256 * 256 - first_byte], len);
        atomicAdd(&nlen[sg.req], len);
    }
}

__global__ void __launch_bounds__(256) nfc_write_kernel(const uint8_t* __restrict__ text, const uint32_t* __restrict__ offsets, uint32_t n,
                                                        uint32_t first_byte, const uint8_t* __restrict__ flags, const uint32_t* __restrict__ tmp_ids,
                                                        const uint32_t* __restrict__ dirty, const uint32_t* __restrict__ seg_len,
                                                        const uint32_t* __restrict__ chunk_sum, const uint8_t* __restrict__ norm_tmp,
                                                        const uint32_t* __restrict__ noff, uint8_t* __restrict__ ntext, uint8_t* __restrict__ nflags,
                                                        uint32_t* __restrict__ nids) {
    __shared__ uint32_t s_w[8];
    const uint32_t r = request_index();
    if (r >= n) return;
    const uint32_t beg = offsets[r], rend = offsets[r + 1];
    const uint32_t cstart = beg + blockIdx.x * blockDim.x;
    if (cstart >= rend) return;
    const uint32_t i = cstart + threadIdx.x;
    const uint32_t out0 = noff[r];
    if (!dirty[r]) {
        if (i < rend) {
            const uint32_t o = out0 + (i - beg);
            const uint8_t fl = flags[i];
            ntext[o] = text[i];
            nflags[o] = fl;
            if (fl >= 2) nids[o] = tmp_ids[i];
        }
        return;
    }
    uint32_t pre = 0;   // output bytes of the request's earlier chunks
    for (uint32_t c = threadIdx.x; c < blockIdx.x; c += blockDim.x) pre += chunk_sum[beg + c * 256 - first_byte];
    const uint32_t base = block_sum_256(pre, s_w);
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const uint32_t len = i < rend ? seg_len[i - first_byte] : 0;
    uint32_t inc = len;   // inclusive scan within the warp, then across the 8 warps
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) { const uint32_t t = __shfl_up_sync(0xffffffffu, inc, d); if (lane >= d) inc += t; }
    if (lane == 31) s_w[wid] = inc;
    __syncthreads();
    uint32_t before = 0;
    for (int w = 0; w < wid; ++w) before += s_w[w];
    if (len) {
        const uint32_t o = out0 + base + before + inc - len;
        const uint8_t fl = flags[i];
        if (fl >= 2) { ntext[o] = text[i]; nflags[o] = fl; nids[o] = tmp_ids[i]; }
        else {
            const uint8_t* src = norm_tmp + 3ull * (i - first_byte);
            for (uint32_t j = 0; j < len; ++j) { ntext[o + j] = src[j]; nflags[o + j] = 0; }
        }
    }
}

// K1m: SentencePiece-style BPE (metaspace.cuh), only for a tokenizer loaded with smgx_tokenizer_load_bpe_metaspace.  Like the NFC stage
// it runs after the specials are resolved on the raw text and writes a normalized ragged copy of the batch (text, flags, the specials'
// ids); a stretch of L raw bytes becomes at most 3L + 3 ≤ 6L bytes and at most L + 1 ≤ 2L initial symbols.  Then:
//   ms_count_kernel      thread per raw byte: output bytes; chunk_sum (per 256-byte chunk) and nlen (per request) collect them
//   scan_counts_kernel   normalized request lengths → offsets of the normalized batch
//   ms_write_kernel      thread per raw byte: writes its bytes at (earlier chunks of the request + exclusive scan within the chunk)
//   ms_symbolize_kernel  thread per normalized byte: a code point's initial symbols into its slots of tmp_ids (ms_symbolize), and flags = 1
//                        where a piece starts (ms_piece_start)
//   ms_emit_kernel       thread per piece start: counts the piece's symbols up to the next start, a special or the request end; a
//                        single symbol is already its token, longer pieces go to the merge kernels' lists by symbol count
// and bpe_merge_kernel<true> / bpe_long_kernel<true> merge them.
__global__ void __launch_bounds__(256) ms_count_kernel(MetaspaceMode mm, const uint8_t* __restrict__ text, const uint32_t* __restrict__ offsets,
                                                       uint32_t n, uint32_t first_byte, const uint8_t* __restrict__ flags,
                                                       uint32_t* __restrict__ chunk_sum, uint32_t* __restrict__ nlen) {
    __shared__ uint32_t s_w[8];
    const uint32_t r = request_index();
    if (r >= n) return;
    const uint32_t beg = offsets[r], rend = offsets[r + 1];
    const uint32_t cstart = beg + blockIdx.x * blockDim.x;
    if (cstart >= rend) return;   // CTA-uniform
    const uint32_t i = cstart + threadIdx.x;
    const uint32_t sum = block_sum_256(i < rend ? ms_out_len(mm, text, flags, i, beg) : 0, s_w);
    if (threadIdx.x == 0) {
        chunk_sum[cstart - first_byte] = sum;
        atomicAdd(&nlen[r], sum);
    }
}

__global__ void __launch_bounds__(256) ms_write_kernel(MetaspaceMode mm, const uint8_t* __restrict__ text, const uint32_t* __restrict__ offsets,
                                                       uint32_t n, uint32_t first_byte, const uint8_t* __restrict__ flags,
                                                       const uint32_t* __restrict__ tmp_ids, const uint32_t* __restrict__ chunk_sum,
                                                       const uint32_t* __restrict__ noff, uint8_t* __restrict__ ntext, uint8_t* __restrict__ nflags,
                                                       uint32_t* __restrict__ nids) {
    __shared__ uint32_t s_w[8];
    const uint32_t r = request_index();
    if (r >= n) return;
    const uint32_t beg = offsets[r], rend = offsets[r + 1];
    const uint32_t cstart = beg + blockIdx.x * blockDim.x;
    if (cstart >= rend) return;
    const uint32_t i = cstart + threadIdx.x;
    uint32_t pre = 0;   // output bytes of the request's earlier chunks
    for (uint32_t c = threadIdx.x; c < blockIdx.x; c += blockDim.x) pre += chunk_sum[beg + c * 256 - first_byte];
    const uint32_t base = block_sum_256(pre, s_w);
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const uint32_t len = i < rend ? ms_out_len(mm, text, flags, i, beg) : 0;
    uint32_t inc = len;   // inclusive scan within the warp, then across the 8 warps
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) { const uint32_t t = __shfl_up_sync(0xffffffffu, inc, d); if (lane >= d) inc += t; }
    if (lane == 31) s_w[wid] = inc;
    __syncthreads();
    uint32_t before = 0;
    for (int w = 0; w < wid; ++w) before += s_w[w];
    if (i < rend) {
        const uint32_t o = noff[r] + base + before + inc - len;
        const uint8_t fl = flags[i];
        ms_out_write(mm, text, flags, i, beg, ntext + o);
        for (uint32_t j = 0; j < len; ++j) nflags[o + j] = fl >= 2 ? fl : 0;
        if (fl >= 2) nids[o] = tmp_ids[i];
    }
}

__global__ void __launch_bounds__(256) ms_symbolize_kernel(BpeView v, uint32_t split, const uint8_t* __restrict__ text, const uint32_t* __restrict__ offsets,
                                                           uint32_t n, uint8_t* __restrict__ flags, uint32_t* __restrict__ tmp_ids) {
    const uint32_t r = request_index();
    if (r >= n) return;
    const uint32_t beg = offsets[r], rend = offsets[r + 1];
    const uint32_t i = beg + blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= rend || flags[i] >= 2 || (text[i] & 0xC0) == 0x80) return;
    uint32_t ns;
    ms_symbolize(v, text, i, rend, tmp_ids + i, &ns);
    if (ms_piece_start(text, flags, i, beg, split)) flags[i] = 1;   // neighbours only test flags >= 2: 0 → 1 does not change their answer
}

__global__ void __launch_bounds__(256) ms_emit_kernel(const uint32_t* __restrict__ offsets, uint32_t n, const uint8_t* __restrict__ flags,
                                                      const uint32_t* __restrict__ tmp_ids, Piece* __restrict__ pieces, uint32_t* __restrict__ counters,
                                                      uint32_t* __restrict__ totals, uint32_t* __restrict__ miss_short, uint32_t* __restrict__ miss_long) {
    const uint32_t r = request_index();
    if (r >= n) return;
    const uint32_t beg = offsets[r], rend = offsets[r + 1];
    const uint32_t cstart = beg + blockIdx.x * blockDim.x;
    if (cstart >= rend) return;   // CTA-uniform: the warps below stay whole
    const uint32_t i = cstart + threadIdx.x;
    const int lane = threadIdx.x & 31;
    uint32_t ns = 0, j = i;
    if (i < rend && flags[i] == 1) {
        for (j = i; j < rend && (j == i || flags[j] == 0); ++j) ns += tmp_ids[j] != kInvalidTok;
    }
    const int kind = ns == 1 ? 3 : ns > kSmemSyms ? 2 : ns ? 1 : 0;   // 3: one symbol, already the token
    const unsigned one = __ballot_sync(0xffffffffu, kind == 3);
    if (lane == 0 && one) atomicAdd(&totals[r], (uint32_t)__popc(one));
#pragma unroll
    for (int k = 1; k <= 2; ++k) {
        const unsigned bal = __ballot_sync(0xffffffffu, kind == k);
        if (!bal) continue;
        const int leader = __ffs((int)bal) - 1;
        uint32_t pbase = 0, lbase = 0;
        if (lane == leader) { pbase = atomicAdd(&counters[0], (uint32_t)__popc(bal)); lbase = atomicAdd(&counters[k], (uint32_t)__popc(bal)); }
        pbase = __shfl_sync(0xffffffffu, pbase, leader);
        lbase = __shfl_sync(0xffffffffu, lbase, leader);
        if (kind == k) {
            const uint32_t rank = (uint32_t)__popc(bal & ((1u << lane) - 1u));
            pieces[pbase + rank] = Piece{i, j - i, r};
            (k == 1 ? miss_short : miss_long)[lbase + rank] = pbase + rank;
        }
    }
}

uint32_t pow2_at_least(uint64_t x) { uint32_t p = 1024; while (p < x) p <<= 1; return p; }

std::string b64decode(const std::string& in) {
    static int8_t T[256];
    static bool init = false;
    if (!init) {
        memset(T, -1, sizeof(T));
        const char* a = "ABCDEFGHIJKLMNOPQRSTUVWXYZabcdefghijklmnopqrstuvwxyz0123456789+/";
        for (int i = 0; i < 64; ++i) T[(uint8_t)a[i]] = (int8_t)i;
        init = true;
    }
    std::string out;
    uint32_t val = 0;
    int bits = -8;
    for (unsigned char c : in) {
        if (c == '=') break;
        if (T[c] < 0) throw Error(SMGX_TOKENIZATION_ERROR, "invalid base64 in tiktoken file");
        val = (val << 6) | (uint32_t)T[c];
        bits += 6;
        if (bits >= 0) { out.push_back((char)((val >> bits) & 0xFF)); bits -= 8; }
    }
    return out;
}

}  // namespace

Tokenizer* Tokenizer::from_tiktoken_file(const std::string& path, const std::vector<std::pair<std::string, uint32_t>>& specials, bool device,
                                          Pretok pretok) {
    // load_tiktoken_bpe (tiktoken.rs:346-367): lines of `base64(token) rank`
    std::ifstream f(path);
    if (!f) throw Error(SMGX_TOKENIZATION_ERROR, "cannot open tiktoken file '" + path + "'");
    std::vector<std::string> toks;
    std::vector<uint32_t> ranks;
    std::string line;
    while (std::getline(f, line)) {
        if (line.empty()) continue;
        std::istringstream ls(line);
        std::string b64, rk;
        if (!(ls >> b64)) throw Error(SMGX_TOKENIZATION_ERROR, "missing token in tiktoken file");
        if (!(ls >> rk)) throw Error(SMGX_TOKENIZATION_ERROR, "missing rank in tiktoken file");
        toks.push_back(b64decode(b64));
        ranks.push_back((uint32_t)std::stoul(rk));
    }
    return new Tokenizer(toks, ranks, specials, device, pretok);
}

Tokenizer::Tokenizer(const std::vector<std::string>& tokens, const std::vector<uint32_t>& ranks,
                     const std::vector<std::pair<std::string, uint32_t>>& specials, bool device, Pretok pretok)
    : device_(device), pretok_(pretok) {
    build(tokens, ranks, nullptr, true, specials);
}
Tokenizer::Tokenizer(const std::vector<std::string>& tokens, const std::vector<uint32_t>& ids, const std::vector<std::pair<uint32_t, uint32_t>>& merges,
                     bool ignore_merges, const std::vector<std::pair<std::string, uint32_t>>& specials, bool device, Pretok pretok, bool nfc)
    : device_(device), pretok_(pretok), nfc_(nfc) {
    build(tokens, ids, &merges, ignore_merges, specials);
}
Tokenizer::Tokenizer(const std::vector<std::string>& tokens, const std::vector<uint32_t>& ids, const std::vector<std::pair<uint32_t, uint32_t>>& merges,
                     const std::vector<std::pair<std::string, uint32_t>>& specials, bool device, MetaspaceMode ms)
    : device_(device), ms_(ms) {
    ms_.on = 1;
    build(tokens, ids, &merges, false, specials);
}

void Tokenizer::build(const std::vector<std::string>& tokens, const std::vector<uint32_t>& ranks, const std::vector<std::pair<uint32_t, uint32_t>>* merges,
                      bool whole_piece, const std::vector<std::pair<std::string, uint32_t>>& specials) {
    SMGX_REQUIRE(tokens.size() == ranks.size() && !tokens.empty(), "empty vocabulary");
    std::unordered_map<std::string, uint32_t> enc;
    enc.reserve(tokens.size() * 2);
    uint32_t max_len = 1, max_id = 0;
    for (size_t i = 0; i < tokens.size(); ++i) {
        SMGX_REQUIRE(!tokens[i].empty(), "empty token in vocabulary");
        enc[tokens[i]] = ranks[i];
        max_len = std::max<uint32_t>(max_len, (uint32_t)tokens[i].size());
        max_id = std::max(max_id, ranks[i]);
    }
    for (auto& sp : specials) max_id = std::max(max_id, sp.second);
    vocab_size_ = max_id + 1;
    SMGX_REQUIRE(vocab_size_ < (1u << 27), "vocabulary too large (merge ranks are packed into 27 bits)");

    std::vector<uint32_t> byte_token(256);
    for (int b = 0; b < 256; ++b) {
        if (ms_.on) {   // byte fallback: `tokenizers` looks up format!("<{b:#04X}>")
            char name[8];
            snprintf(name, sizeof(name), "<0x%02X>", b);
            auto it = enc.find(name);
            if (it == enc.end()) throw Error(SMGX_TOKENIZATION_ERROR, std::string("vocabulary lacks the byte-fallback token ") + name);
            byte_token[b] = it->second;
            continue;
        }
        auto it = enc.find(std::string(1, (char)b));
        if (it == enc.end()) throw Error(SMGX_TOKENIZATION_ERROR, "vocabulary lacks the single-byte token " + std::to_string(b));
        byte_token[b] = it->second;
    }
    static const std::string kMeta = "\xE2\x96\x81";   // ▁
    if (ms_.on && !enc.count(kMeta)) throw Error(SMGX_TOKENIZATION_ERROR, "vocabulary lacks the token \"\xE2\x96\x81\" (U+2581)");
    // blob of token bytes + piece table keyed by the bytes
    std::vector<uint8_t> blob;
    std::vector<PieceSlot> pieces(pow2_at_least(tokens.size() * 2), PieceSlot{0, 0, 0, 0, 0});
    uint32_t pmask = (uint32_t)pieces.size() - 1;
    for (auto& kv : enc) {
        uint32_t off = (uint32_t)blob.size();
        blob.insert(blob.end(), kv.first.begin(), kv.first.end());
        uint64_t hsh = bytes_hash((const uint8_t*)kv.first.data(), (uint32_t)kv.first.size());
        uint32_t h = (uint32_t)(hsh >> 32) & pmask;
        while (pieces[h].hash) h = (h + 1) & pmask;
        pieces[h] = PieceSlot{hsh, kv.second, (uint32_t)kv.first.size(), off, 0};
    }
    // pair table (left id, right id) → (priority, merged id)
    struct PairRec { uint64_t key; uint32_t rank, id; };
    std::vector<PairRec> pair_list;
    if (!merges) {
        // tiktoken: every split of every token into two vocab entries (rank of the concatenation = the merge priority)
        for (auto& kv : enc) {
            const std::string& t = kv.first;
            for (size_t k = 1; k < t.size(); ++k) {
                auto l = enc.find(t.substr(0, k));
                if (l == enc.end()) continue;
                auto r = enc.find(t.substr(k));
                if (r == enc.end()) continue;
                pair_list.push_back({((uint64_t)l->second << 32) | r->second, kv.second, kv.second});
            }
        }
    } else {
        // HuggingFace BPE: only the listed pairs merge, in list order; the merged token is the concatenation (models/bpe/model.rs)
        std::unordered_map<uint32_t, const std::string*> by_id;
        for (auto& kv : enc) by_id[kv.second] = &kv.first;
        for (size_t k = 0; k < merges->size(); ++k) {
            auto l = by_id.find((*merges)[k].first), r = by_id.find((*merges)[k].second);
            if (l == by_id.end() || r == by_id.end()) throw Error(SMGX_TOKENIZATION_ERROR, "merge refers to an unknown token id");
            auto t = enc.find(*l->second + *r->second);
            if (t == enc.end()) throw Error(SMGX_TOKENIZATION_ERROR, "merge result is not in the vocabulary");
            // Pieces are cut before every ▁ that follows another character.  Exact unless a merge joins a symbol that does not end in ▁
            // (a character, or a byte token) to one that starts with ▁: only such a pair can straddle a cut (DESIGN §4c).
            const std::string &ls = *l->second, &rs = *r->second;
            if (ms_.on && !ms_.split && rs.compare(0, kMeta.size(), kMeta) == 0 &&
                !(ls.size() >= kMeta.size() && ls.compare(ls.size() - kMeta.size(), kMeta.size(), kMeta) == 0))
                throw Error(SMGX_TOKENIZATION_ERROR, "merge " + std::to_string(k) + " (\"" + ls + "\", \"" + rs + "\") joins a symbol that does not end "
                            "in \xE2\x96\x81 to one that starts with \xE2\x96\x81: the text cannot be cut into independent pieces at \xE2\x96\x81");
            pair_list.push_back({((uint64_t)l->first << 32) | r->first, (uint32_t)k, t->second});
        }
    }
    n_pairs_ = (uint32_t)pair_list.size();
    std::vector<PairSlot> pairs(pow2_at_least(pair_list.size() * 2 + 2), PairSlot{kPairEmpty, kRankMax, 0});
    uint32_t qmask = (uint32_t)pairs.size() - 1;
    for (auto& pr : pair_list) {
        uint32_t h = (uint32_t)(mix64(pr.key) >> 32) & qmask;
        while (pairs[h].key != kPairEmpty && pairs[h].key != pr.key) h = (h + 1) & qmask;
        if (pairs[h].key == pr.key && pairs[h].rank <= pr.rank) continue;   // a repeated pair keeps its first (best) priority
        pairs[h] = PairSlot{pr.key, pr.rank, pr.id};
    }
    dview_.whole_piece = whole_piece ? 1u : 0u;
    // specials
    std::vector<SpecialTok> sp;
    uint32_t first_bits[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (auto& s : specials) {
        SMGX_REQUIRE(!s.first.empty(), "empty special token");
        uint32_t off = (uint32_t)blob.size();
        blob.insert(blob.end(), s.first.begin(), s.first.end());
        sp.push_back(SpecialTok{off, (uint32_t)s.first.size(), s.second, 0});
        uint8_t c = (uint8_t)s.first[0];
        first_bits[c >> 5] |= 1u << (c & 31);
    }
    if (!device_) return;
    auto up = [](DevBuf& d, const void* src, size_t bytes) {
        d.reserve(std::max<size_t>(bytes, 16));
        if (bytes) SMGX_CUDA(cudaMemcpy(d.ptr, src, bytes, cudaMemcpyHostToDevice));
    };
    up(d_byte_token_, byte_token.data(), 256 * 4);
    up(d_pairs_, pairs.data(), pairs.size() * sizeof(PairSlot));
    up(d_pieces_, pieces.data(), pieces.size() * sizeof(PieceSlot));
    up(d_blob_, blob.data(), blob.size());
    up(d_specials_, sp.data(), sp.size() * sizeof(SpecialTok));
    // the class table of the pre-tokenizer: DeepSeek's chain uses the classes of `tokenizers` (ds_class), the other patterns char_class
    const bool ds = pretok_ == Pretok::DeepSeek;
    up(d_uni_lo_, ds ? kDsLo : kUniLo, ds ? sizeof(kDsLo) : sizeof(kUniLo));
    up(d_uni_hi_, ds ? kDsHi : kUniHi, ds ? sizeof(kDsHi) : sizeof(kUniHi));
    up(d_uni_cls_, ds ? kDsCls : kUniCls, ds ? sizeof(kDsCls) : sizeof(kUniCls));
    dview_.byte_token = d_byte_token_.as<uint32_t>();
    dview_.pairs = d_pairs_.as<PairSlot>();
    dview_.pair_mask = qmask;
    dview_.pieces = d_pieces_.as<PieceSlot>();
    dview_.piece_mask = pmask;
    dview_.blob = d_blob_.as<uint8_t>();
    dview_.max_token_len = max_len;
    dview_.specials = d_specials_.as<SpecialTok>();
    dview_.n_special = (uint32_t)sp.size();
    for (int i = 0; i < 8; ++i) dview_.special_first[i] = first_bits[i];
    dview_.uni = UnicodeView{d_uni_lo_.as<uint32_t>(), d_uni_hi_.as<uint32_t>(), d_uni_cls_.as<uint8_t>(), ds ? kDsRanges : kUniRanges};
    if (nfc_) {   // the NFC tables, one allocation (every array 16-byte aligned)
        std::vector<uint8_t> t;
        auto put = [&t](const void* src, size_t bytes) {
            const size_t at = (t.size() + 15) / 16 * 16;
            t.resize(at + bytes);
            memcpy(t.data() + at, src, bytes);
            return at;
        };
        const size_t o_ccp = put(kNfcCccCp, sizeof(kNfcCccCp)), o_cv = put(kNfcCccVal, sizeof(kNfcCccVal));
        const size_t o_dcp = put(kNfcDecCp, sizeof(kNfcDecCp)), o_doff = put(kNfcDecOff, sizeof(kNfcDecOff)), o_dd = put(kNfcDecData, sizeof(kNfcDecData));
        const size_t o_ck = put(kNfcCompKey, sizeof(kNfcCompKey)), o_cval = put(kNfcCompVal, sizeof(kNfcCompVal));
        const size_t o_ulo = put(kNfcUnstLo, sizeof(kNfcUnstLo)), o_uhi = put(kNfcUnstHi, sizeof(kNfcUnstHi));
        up(d_nfc_, t.data(), t.size());
        const uint8_t* b = d_nfc_.as<uint8_t>();
        nview_ = NfcView{(const uint32_t*)(b + o_ccp), b + o_cv, kNfcCccN, (const uint32_t*)(b + o_dcp), (const uint16_t*)(b + o_doff),
                         (const uint32_t*)(b + o_dd), kNfcDecN, (const uint64_t*)(b + o_ck), (const uint32_t*)(b + o_cval), kNfcCompN,
                         (const uint32_t*)(b + o_ulo), (const uint32_t*)(b + o_uhi), kNfcUnstableN};
    }
}

Tokenizer::~Tokenizer() {
    d_byte_token_.release(); d_pairs_.release(); d_pieces_.release(); d_blob_.release(); d_specials_.release();
    d_uni_lo_.release(); d_uni_hi_.release(); d_uni_cls_.release(); d_nfc_.release();
}

void Tokenizer::encode_batch(const uint8_t* d_text, const uint32_t* d_offsets, uint32_t n, uint32_t first_byte, uint32_t total_bytes, uint32_t max_len,
                             uint32_t* d_tokens, uint32_t* d_tok_offsets, Scratch& sc, cudaStream_t stream, uint64_t* launches) const {
    if (!device_) throw Error(SMGX_DEVICE_ERROR, "tokenizer was loaded without a device (host-mirror policy): no GPU path, no CPU fallback");
    if (n == 0) return;
    const uint32_t raw = total_bytes - first_byte;
    const bool norm = nfc_ || ms_.on;
    const uint64_t tg = text_growth();
    if (norm) SMGX_REQUIRE(tg * raw < (1ull << 31) && tg * max_len < (1ull << 31), "text batch too large for the normalizer");
    // bytes the pre-tokenizer and BPE see: the raw text, or its normalized copy (at most text_growth() times as long, at absolute
    // offsets from 0)
    const uint32_t span = norm ? (uint32_t)(tg * raw) : raw;
    const uint32_t span_end = norm ? span : total_bytes;
    sc.flags.reserve(std::max<uint32_t>(total_bytes, 1));
    sc.tmp_ids.reserve((size_t)std::max<uint32_t>(total_bytes, 1) * 4);
    sc.tmp_rk.reserve((size_t)std::max<uint32_t>(std::max(total_bytes, span_end), 1) * 8);
    sc.totals.reserve((size_t)n * 4);
    sc.pieces.reserve((size_t)std::max<uint32_t>(span, 1) * sizeof(Piece));
    sc.n_pieces.reserve(16);
    sc.miss.reserve(((size_t)std::max<uint32_t>(span, 1) + 1) * 8);
    if (total_bytes) {
        SMGX_CUDA(cudaMemsetAsync(sc.flags.ptr, 0, total_bytes, stream));
    }
    {
        const dim3 grid2 = request_grid((max_len + 255) / 256, n);
        if (dview_.n_special && max_len) {
            special_candidates_kernel<<<grid2, 256, 0, stream>>>(dview_, d_text, d_offsets, n, sc.flags.as<uint8_t>(), sc.tmp_ids.as<uint32_t>(),
                                                               sc.tmp_rk.as<uint64_t>());
            SMGX_CUDA(cudaGetLastError());
            ++*launches;
            special_resolve_kernel<<<(unsigned)(((uint64_t)n * 32 + 255) / 256), 256, 0, stream>>>(d_offsets, n, sc.flags.as<uint8_t>(), sc.tmp_ids.as<uint32_t>(),
                                                                                               sc.tmp_rk.as<uint64_t>(), sc.totals.as<uint32_t>());
            SMGX_CUDA(cudaGetLastError());
            ++*launches;
        } else {
            SMGX_CUDA(cudaMemsetAsync(sc.totals.ptr, 0, (size_t)n * 4, stream));
        }
        // what the pre-tokenizer, BPE and compaction run on
        const uint8_t* text = d_text;
        const uint32_t* offsets = d_offsets;
        uint8_t* flags = sc.flags.as<uint8_t>();
        uint32_t* tmp_ids = sc.tmp_ids.as<uint32_t>();
        uint32_t len_bound = max_len;
        if (nfc_ && max_len) {
            // scratch, 16-byte aligned slices of one allocation: normalized text / flags / ids (3 per raw byte), segment lengths and
            // chunk sums (per raw byte), segment output (3 bytes per raw byte), long-segment entries (4 per raw byte), the long list,
            // and per request: dirty, normalized length, normalized offsets; then the long count
            const size_t R = std::max<uint32_t>(raw, 1);
            size_t at = 0;
            auto slice = [&at](size_t bytes) { const size_t o = at; at = (at + bytes + 15) / 16 * 16; return o; };
            const size_t o_text = slice(3 * R), o_flags = slice(3 * R), o_ids = slice(3 * R * 4), o_seg = slice(R * 4), o_chunk = slice(R * 4),
                         o_tmp = slice(3 * R), o_ent = slice(4 * R * 4), o_long = slice((R / 16 + 1) * sizeof(NfcLong)), o_req = slice(((size_t)3 * n + 1) * 4),
                         o_cnt = slice(16);
            sc.nfc.reserve(at);
            uint8_t* b = sc.nfc.as<uint8_t>();
            uint32_t* dirty = (uint32_t*)(b + o_req);
            uint32_t* nlen = dirty + n;
            uint32_t* noff = nlen + n;
            uint32_t* n_long = (uint32_t*)(b + o_cnt);
            SMGX_CUDA(cudaMemsetAsync(dirty, 0, (size_t)n * 8, stream));   // dirty and nlen
            SMGX_CUDA(cudaMemsetAsync(n_long, 0, 16, stream));
            // the raw-coordinate arrays are indexed from first_byte
            uint32_t* seg_len = (uint32_t*)(b + o_seg);
            uint32_t* chunk_sum = (uint32_t*)(b + o_chunk);
            uint8_t* norm_tmp = b + o_tmp;
            NfcLong* longs = (NfcLong*)(b + o_long);
            nfc_check_kernel<<<grid2, 256, 0, stream>>>(nview_, d_text, d_offsets, n, flags, dirty);
            nfc_segment_kernel<<<grid2, 256, 0, stream>>>(nview_, d_text, d_offsets, n, first_byte, flags, dirty, seg_len, chunk_sum, nlen, norm_tmp, longs,
                                                          n_long);
            const unsigned sms = current_sm_count();
            nfc_long_kernel<<<sms, 256, 0, stream>>>(nview_, d_text, d_offsets, first_byte, longs, n_long, (uint32_t*)(b + o_ent), seg_len, chunk_sum, nlen, norm_tmp);
            scan_counts_kernel<<<1, 1024, 0, stream>>>(nlen, n, noff);
            nfc_write_kernel<<<grid2, 256, 0, stream>>>(d_text, d_offsets, n, first_byte, flags, tmp_ids, dirty, seg_len, chunk_sum, norm_tmp, noff,
                                                        b + o_text, b + o_flags, (uint32_t*)(b + o_ids));
            SMGX_CUDA(cudaGetLastError());
            *launches += 5;
            text = b + o_text;
            offsets = noff;
            flags = b + o_flags;
            tmp_ids = (uint32_t*)(b + o_ids);
            len_bound = 3 * max_len;
        } else if (ms_.on && max_len) {
            // scratch, 16-byte aligned slices of one allocation: normalized text / flags / ids (6 per raw byte), chunk sums (per raw
            // byte), per request: normalized length and offsets
            const size_t R = std::max<uint32_t>(raw, 1);
            size_t at = 0;
            auto slice = [&at](size_t bytes) { const size_t o = at; at = (at + bytes + 15) / 16 * 16; return o; };
            const size_t o_text = slice(6 * R), o_flags = slice(6 * R), o_ids = slice(6 * R * 4), o_chunk = slice(R * 4),
                         o_req = slice(((size_t)2 * n + 1) * 4);
            sc.nfc.reserve(at);
            uint8_t* b = sc.nfc.as<uint8_t>();
            uint32_t* nlen = (uint32_t*)(b + o_req);
            uint32_t* noff = nlen + n;
            uint32_t* chunk_sum = (uint32_t*)(b + o_chunk);   // indexed from first_byte
            SMGX_CUDA(cudaMemsetAsync(nlen, 0, (size_t)n * 4, stream));
            ms_count_kernel<<<grid2, 256, 0, stream>>>(ms_, d_text, d_offsets, n, first_byte, flags, chunk_sum, nlen);
            scan_counts_kernel<<<1, 1024, 0, stream>>>(nlen, n, noff);
            ms_write_kernel<<<grid2, 256, 0, stream>>>(ms_, d_text, d_offsets, n, first_byte, flags, tmp_ids, chunk_sum, noff, b + o_text, b + o_flags,
                                                       (uint32_t*)(b + o_ids));
            SMGX_CUDA(cudaGetLastError());
            *launches += 3;
            text = b + o_text;
            offsets = noff;
            flags = b + o_flags;
            tmp_ids = (uint32_t*)(b + o_ids);
            len_bound = 6 * max_len;
        }
        SMGX_CUDA(cudaMemsetAsync(sc.n_pieces.ptr, 0, 16, stream));
        if (max_len && ms_.on) {
            // segmenter + symbolizer instead of the pre-tokenizer and the whole-piece lookup, then the merge tiers by symbol count
            const dim3 gridn = request_grid((len_bound + 255) / 256, n);   // CTAs past a request's normalized end return at once
            const unsigned sms = current_sm_count();
            const unsigned grid = (unsigned)std::min<uint64_t>(((uint64_t)span / 2 + 255) / 256 + 1, sms * 16ull);
            uint32_t* cnt = sc.n_pieces.as<uint32_t>();
            uint32_t* miss_short = sc.miss.as<uint32_t>();
            uint32_t* miss_long = miss_short + span + 1;
            ms_symbolize_kernel<<<gridn, 256, 0, stream>>>(dview_, ms_.split, text, offsets, n, flags, tmp_ids);
            ms_emit_kernel<<<gridn, 256, 0, stream>>>(offsets, n, flags, tmp_ids, sc.pieces.as<Piece>(), cnt, sc.totals.as<uint32_t>(), miss_short, miss_long);
            bpe_merge_kernel<true><<<std::min(grid, sms * 4), 256, 0, stream>>>(dview_, text, sc.pieces.as<Piece>(), cnt, miss_short, tmp_ids, sc.totals.as<uint32_t>());
            bpe_long_kernel<true><<<std::min(grid, sms * 8), 256, 0, stream>>>(dview_, text, sc.pieces.as<Piece>(), cnt, miss_long, tmp_ids,
                                                                          sc.tmp_rk.as<uint64_t>(), sc.totals.as<uint32_t>());
            SMGX_CUDA(cudaGetLastError());
            *launches += 4;
        } else if (max_len) {
            const dim3 gridp = request_grid((len_bound + 255) / 256, n);   // with NFC: CTAs past a request's normalized end find an empty window
            if (pretok_ == Pretok::R50k)
                pretokenize_kernel<Pretok::R50k><<<gridp, 256, 0, stream>>>(dview_, text, offsets, n, flags, sc.pieces.as<Piece>(), sc.n_pieces.as<uint32_t>());
            else if (pretok_ == Pretok::Qwen2)
                pretokenize_kernel<Pretok::Qwen2><<<gridp, 256, 0, stream>>>(dview_, text, offsets, n, flags, sc.pieces.as<Piece>(), sc.n_pieces.as<uint32_t>());
            else if (pretok_ == Pretok::DeepSeek)
                pretokenize_kernel<Pretok::DeepSeek><<<gridp, 256, 0, stream>>>(dview_, text, offsets, n, flags, sc.pieces.as<Piece>(),
                                                                                sc.n_pieces.as<uint32_t>());
            else
                pretokenize_kernel<Pretok::Cl100k><<<gridp, 256, 0, stream>>>(dview_, text, offsets, n, flags, sc.pieces.as<Piece>(), sc.n_pieces.as<uint32_t>());
            SMGX_CUDA(cudaGetLastError());
            ++*launches;
            // the piece count lives on the device, so the grids are sized for the worst case the text allows and stride over the lists
            const unsigned sms = current_sm_count();
            const unsigned grid = (unsigned)std::min<uint64_t>(((uint64_t)span / 2 + 255) / 256 + 1, sms * 16ull);
            uint32_t* cnt = sc.n_pieces.as<uint32_t>();
            uint32_t* miss_short = sc.miss.as<uint32_t>();
            uint32_t* miss_long = miss_short + span + 1;
            bpe_lookup_kernel<<<grid, 256, 0, stream>>>(dview_, text, sc.pieces.as<Piece>(), cnt, tmp_ids, sc.totals.as<uint32_t>(), miss_short, miss_long);
            bpe_merge_kernel<false><<<std::min(grid, sms * 4), 256, 0, stream>>>(dview_, text, sc.pieces.as<Piece>(), cnt, miss_short, tmp_ids, sc.totals.as<uint32_t>());
            bpe_long_kernel<false><<<std::min(grid, sms * 8), 256, 0, stream>>>(dview_, text, sc.pieces.as<Piece>(), cnt, miss_long, tmp_ids,
                                                                           sc.tmp_rk.as<uint64_t>(), sc.totals.as<uint32_t>());
            SMGX_CUDA(cudaGetLastError());
            *launches += 3;
        }
        scan_counts_kernel<<<1, 1024, 0, stream>>>(sc.totals.as<uint32_t>(), n, d_tok_offsets);
        SMGX_CUDA(cudaGetLastError());
        ++*launches;
        compact_tokens_kernel<<<(unsigned)(((uint64_t)n * 32 + 255) / 256), 256, 0, stream>>>(offsets, n, tmp_ids, d_tok_offsets, d_tokens);
        SMGX_CUDA(cudaGetLastError());
        ++*launches;
    }
}

}  // namespace smgx
