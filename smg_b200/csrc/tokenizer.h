// K1 — GPU tokenizer (tiktoken-style BPE): vocabulary tables on the device + the batch tokenize launch.
// Host-side counterpart of TiktokenTokenizer (crates/tokenizer/src/tiktoken.rs:132-462): load_tiktoken_bpe (:346-367),
// the special-token encoder (:234-238) and encode → CoreBPE::encode_with_special_tokens (:444-462).
#pragma once
#include <cstdint>
#include <string>
#include <vector>

#include "bpe.cuh"
#include "common.h"
#include "metaspace.cuh"
#include "nfc.cuh"

namespace smgx {

class Tokenizer {
public:
    // tokens[i] = bytes of the vocab entry with rank/id ranks[i]; specials = (string, id); pretok = the pre-tokenizer regex
    Tokenizer(const std::vector<std::string>& tokens, const std::vector<uint32_t>& ranks,
              const std::vector<std::pair<std::string, uint32_t>>& specials, bool device, Pretok pretok);
    // HuggingFace `tokenizers` BPE (byte-level): merge priority = position in `merges` (pairs of ids), only listed pairs merge;
    // ignore_merges = look the whole piece up in the vocabulary first (models::bpe ignore_merges, Llama 3).
    // nfc: the tokenizer.json normalizer is NFC (nfc.cuh); the text between specials is normalized before it is split.
    Tokenizer(const std::vector<std::string>& tokens, const std::vector<uint32_t>& ids, const std::vector<std::pair<uint32_t, uint32_t>>& merges,
              bool ignore_merges, const std::vector<std::pair<std::string, uint32_t>>& specials, bool device, Pretok pretok, bool nfc = false);
    // SentencePiece-style BPE with byte fallback (metaspace.cuh): tokens are raw UTF-8 strings, the byte-fallback tokens are the vocabulary
    // entries "<0x00>" … "<0xFF>"; `ms` says how spaces become ▁ and where pieces start.  Refuses (SMGX_TOKENIZATION_ERROR) a vocabulary
    // without ▁ or one of the byte tokens, and — when pieces are cut only at ▁ after another character — a merge that could join
    // two pieces (DESIGN §4c).
    Tokenizer(const std::vector<std::string>& tokens, const std::vector<uint32_t>& ids, const std::vector<std::pair<uint32_t, uint32_t>>& merges,
              const std::vector<std::pair<std::string, uint32_t>>& specials, bool device, MetaspaceMode ms);
    ~Tokenizer();
    static Tokenizer* from_tiktoken_file(const std::string& path, const std::vector<std::pair<std::string, uint32_t>>& specials, bool device,
                                         Pretok pretok);

    BpeView view() const { return dview_; }
    uint32_t vocab_size() const { return vocab_size_; }
    uint32_t n_pairs() const { return n_pairs_; }
    // Most tokens per byte of input: 3 with NFC (U+1D160 → three code points), 2 for SentencePiece-style BPE (a stretch of L bytes has at
    // most L + 1 initial symbols), else 1.
    uint32_t growth() const { return nfc_ ? 3u : ms_.on ? 2u : 1u; }
    // Most bytes of normalized text per byte of input: 3 with NFC, 6 for SentencePiece-style BPE (" " → "▁▁" at a stretch start), else 1.
    uint32_t text_growth() const { return nfc_ ? 3u : ms_.on ? 6u : 1u; }

    // Scratch needed for a batch of `total_bytes` of text and `n` requests; `nfc` holds the normalization stage's buffers (NFC or ▁).
    struct Scratch { DevBuf flags, tmp_ids, tmp_rk, totals, pieces, n_pieces, miss, nfc; };

    // Enqueue [NFC or ▁ normalization +] pre-tokenise + BPE + compaction on `stream`.
    //   d_text/d_offsets (n+1): ragged UTF-8; d_tokens: capacity ≥ growth() × (total_bytes - first_byte) u32; d_tok_offsets: n+1 u32 (written).
    // Text bytes live at d_text[first_byte .. total_bytes) (absolute offsets as given in d_offsets).
    // `max_len` = longest request in bytes (sizes the 2-D grids).
    void encode_batch(const uint8_t* d_text, const uint32_t* d_offsets, uint32_t n, uint32_t first_byte, uint32_t total_bytes, uint32_t max_len,
                      uint32_t* d_tokens, uint32_t* d_tok_offsets, Scratch& sc, cudaStream_t stream, uint64_t* launches) const;

private:
    void build(const std::vector<std::string>& tokens, const std::vector<uint32_t>& ranks, const std::vector<std::pair<uint32_t, uint32_t>>* merges,
               bool whole_piece, const std::vector<std::pair<std::string, uint32_t>>& specials);
    BpeView dview_{};
    uint32_t vocab_size_ = 0, n_pairs_ = 0;
    bool device_ = false;
    Pretok pretok_ = Pretok::Cl100k;
    bool nfc_ = false;
    MetaspaceMode ms_{};
    NfcView nview_{};
    DevBuf d_byte_token_, d_pairs_, d_pieces_, d_blob_, d_specials_, d_uni_lo_, d_uni_hi_, d_uni_cls_, d_nfc_;
};

}  // namespace smgx
