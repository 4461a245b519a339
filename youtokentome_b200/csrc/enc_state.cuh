// enc_state.cuh — the opened model on the device (struct yttm_enc), shared by encode.cu and decode.cu.
#pragma once
#include <string>
#include <vector>

#include "common.cuh"

struct yttm_dec;  // decode state (decode.cu): piece table + per-call buffers, made by the first decode call
void yttm_dec_free(yttm_dec *d);
struct yttm_enc;
// The piece of every id in [0, vocab) as id_to_subword gives it (recipe UTF-8 with a leading U+2581 kept, special ids
// their token); special[i] = 1 for the special ids.  Checks the model tables; error texts start with `who`.
int yttm_model_pieces(yttm_enc *e, const char *who, std::vector<std::string> *raw, std::vector<uint8_t> *special);
// The checks every encode and decode entry point makes before it runs (encode.cu): a handle, its device made current,
// and a model with <BOS> / <EOS> when they are asked for.  Returns 1 with the error recorded (a null handle's text
// starts with `who`).
int yttm_enc_check(yttm_enc *e, const char *who, int bos, int eos);

struct yttm_enc {
  yttm_ctx *ctx = nullptr;
  ytc::DevBuf cp2id, rules;
  uint32_t rule_mask = 0, space_id = 0;
  int unk = -1, pad = -1, bos = -1, eos = -1;
  // host copies of the model tables as yttm_enc_create received them: decode builds its piece table from them
  std::vector<uint32_t> h_char_cp, h_char_id, h_rules_xyz;
  uint64_t vocab = 0;  // n_chars + n_rules + special tokens, BaseEncoder::vocab_size
  yttm_dec *dec = nullptr;
  // spans / subwords (encode.cu), built by their first call: piece_off u32[V+1] | units u32[V] | piece bytes.
  // units[i] = code points of id i's recipe without a leading U+2581: the valid units of a word an id covers.
  ytc::DevBuf sub_table;
  const uint32_t *sub_piece_off = nullptr, *sub_units = nullptr;
  const uint8_t *sub_bytes = nullptr;
  // per-call device buffers: two sets, so that the host-buffer entry point can pipeline chunks
  // (H2D of chunk i+1 and D2H of chunk i-1 overlap the kernels of chunk i)
  struct Slot {
    ytc::DevBuf d_bytes, d_offs, slots, ranks, aux, wpos, wsent, lookback, out_off, out_ids, counter, longw;
    ytc::DevBuf dd_tab, dd_rep, dd_list;  // word dedup
    ytc::DevBuf swb, swc, rec;             // per-sentence word ranges, per-word records (id count, first ids)
    ytc::DevBuf rel, out_spans;            // spans: per-slot span relative to the word start, (start, end) per id
    ytc::DevBuf sub_len, sub_off, sub_out; // subwords: piece length per id, piece offsets, piece bytes
    void release() {
      ytc::DevBuf *b[] = {&d_bytes, &d_offs, &slots, &ranks, &aux, &wpos, &wsent, &lookback, &out_off, &out_ids, &counter, &longw,
                          &dd_tab, &dd_rep, &dd_list, &swb, &swc, &rec, &rel, &out_spans, &sub_len, &sub_off, &sub_out};
      for (auto *x : b) x->release();
    }
  } slot[2];
  cudaStream_t s_in = nullptr, s_out = nullptr;
  cudaEvent_t ev_in[2] = {nullptr, nullptr}, ev_done[2] = {nullptr, nullptr}, ev_out[2] = {nullptr, nullptr};
};
