// enc_state.cuh — the opened model on the device (struct yttm_enc), shared by encode.cu and decode.cu.
#pragma once
#include <string>
#include <vector>

#include "common.cuh"

struct yttm_enc_stream;  // an open encode stream (encode.cu, yttm_enc_stream_*)
void yttm_enc_stream_free(yttm_enc_stream *s);
struct yttm_dec_stream;  // an open decode stream (decode.cu, yttm_dec_stream_*)
void yttm_dec_stream_free(yttm_dec_stream *s);
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
    ytc::DevBuf d_bytes, d_offs, slots, ranks, aux, wpos, wsent, wlen, lookback, out_off, out_ids, counter, longw;
    ytc::DevBuf dd_tab, dd_rep, dd_list;  // word dedup
    ytc::DevBuf swb, swc, rec;             // per-sentence word ranges, per-word records (id count, first ids)
    ytc::DevBuf rel, out_spans;            // spans: per-slot span relative to the word start, (start, end) per id
    ytc::DevBuf sub_len, sub_off, sub_out; // subwords: piece length per id, piece offsets, piece bytes
    // windows (the packed output above is their source): rows per sentence, row bases, then the rows and per row
    // its length, sentence and start
    ytc::DevBuf win_cnt, win_base, win_ids, win_spans, win_len, win_sent, win_start;
    template <class F> void each(F f) {
      ytc::DevBuf *b[] = {&d_bytes, &d_offs, &slots, &ranks, &aux, &wpos, &wsent, &wlen, &lookback, &out_off, &out_ids, &counter, &longw,
                          &dd_tab, &dd_rep, &dd_list, &swb, &swc, &rec, &rel, &out_spans, &sub_len, &sub_off, &sub_out,
                          &win_cnt, &win_base, &win_ids, &win_spans, &win_len, &win_sent, &win_start};
      for (auto *x : b) f(x);
    }
    void release() { each([](ytc::DevBuf *x) { x->release(); }); }
  } slot[2];
  cudaStream_t s_in = nullptr, s_out = nullptr;
  cudaEvent_t ev_in[2] = {nullptr, nullptr}, ev_done[2] = {nullptr, nullptr}, ev_out[2] = {nullptr, nullptr};
  yttm_enc_stream *stream = nullptr;  // open between yttm_enc_stream_begin and _end; owns both slots meanwhile
  yttm_dec_stream *dec_stream = nullptr;  // open between yttm_dec_stream_begin and _end; owns s_in / s_out meanwhile
};

// The host side of the encode and decode streams (encode.cu).  Fed input is staged in two pinned buffers and cut into
// pieces; piece i is copied into *dev_in[i & 1] on the encoder's s_in while piece i - 1 runs its kernels on the context
// stream and piece i - 2 is copied out on s_out and handed to the sink, on the caller's thread, in order.
struct yttm_piece_pipe {
  yttm_enc *e = nullptr;
  uint64_t piece = 0;  // nominal piece bytes
  // 0: text, cut behind the last '\n' of the staged bytes (yttm_pipe_feed_text); else the bytes of one id, fed in whole
  // lines with their ends (yttm_pipe_feed_lines): the piece is its ids, then from (ids bytes + 15) & ~15 its
  // n_lines + 1 line ends as global id counts (the first: the ids before the piece)
  uint32_t unit = 0;
  ytc::DevBuf *dev_in[2] = {nullptr, nullptr};  // the device copy of the piece in slot s (16 spare bytes)
  // The kernels of the piece in slot s (pc[s]: n_bytes and n_lines of an id piece, open_end of a text piece): sets
  // pc[s].n_lines and pc[s].n_out, *data (n_out bytes for the sink) and *ends (n_lines line ends for the sink).
  int (*run)(void *owner, int s, const void **data, const unsigned long long **ends) = nullptr;
  void *owner = nullptr;
  yttm_enc_sink sink = nullptr;
  void *user = nullptr;
  const char *who = "";                     // the stream's name in error texts
  uint8_t *stage[2] = {nullptr, nullptr};   // pinned staging of the fed bytes: piece i is copied in from stage[i & 1]
  uint64_t stage_cap[2] = {0, 0};
  uint8_t *ends[2] = {nullptr, nullptr};    // id pieces: their staged line ends (uint64)
  uint64_t ends_cap[2] = {0, 0};
  int cur = 0;                              // staging buffer being filled
  uint64_t len = 0, nonl = 0;               // its bytes; its first bytes known to hold no '\n'
  uint64_t n_ends = 0;                      // id pieces: its lines
  uint8_t *out[2] = {nullptr, nullptr};     // pinned results of the piece in slot s: data, then its line ends
  uint64_t out_cap[2] = {0, 0};
  struct Piece {
    uint64_t n_bytes = 0, n_lines = 0, n_out = 0;
    uint64_t first_id = 0;                  // id pieces: the ids fed before the piece
    bool open_end = false;                  // the last line has no '\n' (the end of the stream)
  } pc[2];
  int to_run = -1, to_deliver = -1;         // slot copied in, not yet run; slot copied out, not yet given to the sink
  uint64_t bytes_in = 0, ids_in = 0;        // fed bytes; id pieces: fed ids
};
// The copy streams and events of the two slots (made by the first call that pipelines).
int yttm_pipe_init(yttm_enc *e);
int yttm_pipe_feed_text(yttm_piece_pipe *p, const char *bytes, uint64_t n);
// whole lines: ids (n_ids of p->unit bytes) and their ends as global id counts, checked by the caller
int yttm_pipe_feed_lines(yttm_piece_pipe *p, const void *ids, uint64_t n_ids, const uint64_t *line_ends, uint64_t n_lines);
// runs what is left and hands it to the sink
int yttm_pipe_end(yttm_piece_pipe *p);
// waits for the encoder's streams and frees the pinned buffers
void yttm_pipe_free(yttm_piece_pipe *p);
// The lines of the n bytes at d (device): *n_lines of them, offsets (n_lines + 1: 0, the byte behind every '\n', n when
// open_end) in offs; tiles is scratch.  One 8-byte read-back.
int yttm_line_split(yttm_ctx *c, const uint8_t *d, uint64_t n, bool open_end, ytc::DevBuf *tiles, ytc::DevBuf *offs,
                    uint64_t *n_lines);
// off[0, n) += base on the context stream
void yttm_add_base(yttm_ctx *c, unsigned long long *off, uint64_t n, unsigned long long base);
