// capi.cpp — flat C entry points over the host C++ surface (bpe_b200.h) for the Python package
// (youtokentome_b200/_lib.py binds them with ctypes; it plays the role of the reference's
// Cython module youtokentome/cpp/yttm.pyx).  Strings are UTF-8; errors come back as
// (non-zero return, message in the handle / thread-local buffer).
#include <cstring>
#include <mutex>
#include <string>
#include <unordered_set>
#include <vector>

#include "../../include/bpe_b200.h"
#include "../../include/yttm_b200_api.h"

using namespace vkcom;

namespace {
thread_local std::string g_err;
// Results of the two-call entry points live in THREAD-LOCAL storage, so two host threads that share one handle (ctypes
// releases the GIL during foreign calls; the reference's Cython module does not) can never read each other's result or
// overrun a buffer sized for another thread's total.  The encoder itself keeps mutable device state (double-buffered
// per-call device buffers, the dropout sentence counter): every call that runs kernels holds the handle's mutex.
struct Result {
  std::vector<int32_t> ids;
  std::vector<uint64_t> offs;
  std::string text;                 // pieces back to back, no separators
  std::vector<uint64_t> piece_off;  // n_pieces + 1 byte offsets into text
  std::vector<uint64_t> sent_off;   // n_sentences + 1 piece indices
  void clear_text() { text.clear(); piece_off.assign(1, 0); sent_off.assign(1, 0); }
  void add_piece(const std::string &p) { text += p; piece_off.push_back(text.size()); }
  void end_sentence() { sent_off.push_back(piece_off.size() - 1); }
};
thread_local Result g_res;
struct Handle {
  BaseEncoder *enc = nullptr;
  std::string err;
  std::mutex mu;
};
int fail(Handle *h, const std::string &m) { (h ? h->err : g_err) = m; return 1; }
// the return code of a call that reports a Status: 0, 1 (error, message in the handle) or 2 (a caller buffer too small:
// the counts hold the sizes needed, nothing written)
int ret(Handle *h, const Status &st) { return st.code == 2 ? 2 : st.ok() ? 0 : fail(h, st.message); }
}  // namespace

extern "C" {

const char *yttm_api_last_error(void *hv) { return hv ? static_cast<Handle *>(hv)->err.c_str() : g_err.c_str(); }

int yttm_api_train(const char *data_path, const char *model_path, int vocab_size, double coverage, int n_threads,
                   int pad_id, int unk_id, int bos_id, int eos_id) {
  BpeConfig cfg(coverage, n_threads, SpecialTokens(pad_id, unk_id, bos_id, eos_id));
  Status st = train_bpe(data_path, model_path, vocab_size, cfg);
  if (!st.ok()) return fail(nullptr, st.message);
  return 0;
}

int yttm_api_train_memory(const char *text, uint64_t n, const char *model_path, int vocab_size, double coverage,
                          int pad_id, int unk_id, int bos_id, int eos_id) {
  BpeConfig cfg(coverage, 1, SpecialTokens(pad_id, unk_id, bos_id, eos_id));
  std::string data(text, text + n);
  BPEState state;
  Status st = learn_bpe_from_string(data, vocab_size, model_path ? model_path : "", cfg, &state);
  if (!st.ok()) return fail(nullptr, st.message);
  return 0;
}

thread_local WordCounts g_counts;   // the table of the last yttm_api_count_words of this thread

int yttm_api_count_words(int in_fd, const char *text, uint64_t n, const char *tsv_path, uint64_t *sizes) {
  Status st = count_words(in_fd, text, n, tsv_path ? tsv_path : "", &g_counts);
  if (!st.ok()) { g_counts = WordCounts(); return fail(nullptr, st.message); }
  sizes[0] = g_counts.counts.size();
  sizes[1] = g_counts.bytes.size();
  sizes[2] = g_counts.separators;
  sizes[3] = g_counts.data_len;
  return 0;
}

void yttm_api_result_words(uint8_t *bytes, uint64_t *offsets, uint64_t *counts) {
  std::memcpy(bytes, g_counts.bytes.data(), g_counts.bytes.size());
  std::memcpy(offsets, g_counts.offsets.data(), g_counts.offsets.size() * 8);
  std::memcpy(counts, g_counts.counts.data(), g_counts.counts.size() * 8);
  g_counts = WordCounts();
}

int yttm_api_train_counts(const uint8_t *bytes, const uint64_t *offsets, const uint64_t *counts, uint64_t n,
                          uint64_t separators, int on_device, const char *tsv_path, const char *model_path,
                          int vocab_size, double coverage, int n_threads, int pad_id, int unk_id, int bos_id,
                          int eos_id) {
  CountsInput in;
  in.bytes = bytes; in.offsets = offsets; in.counts = counts; in.n = n; in.separators = separators;
  in.on_device = on_device;
  in.tsv_path = tsv_path ? tsv_path : "";
  BpeConfig cfg(coverage, n_threads, SpecialTokens(pad_id, unk_id, bos_id, eos_id));
  Status st = train_counts(in, model_path, vocab_size, cfg);
  if (!st.ok()) return fail(nullptr, st.message);
  return 0;
}

void yttm_api_release_training_cache(void) { release_training_cache(); }
int yttm_api_training_cache_held(void) { return training_cache_held(); }

int yttm_api_train_report(double *out, int n) {
  const TrainReport &r = last_train_report();
  double v[] = {(double)r.n_bytes, (double)r.data_len, (double)r.n_words, (double)r.n_unique, (double)r.n_tokens,
                (double)r.n_pairs, (double)r.n_merges, r.read_s, r.h2d_ms, r.char_hist_ms, r.word_count_ms,
                r.tokenise_ms, r.pair_hist_ms, r.merge_loop_ms, r.total_s, (double)r.launches, (double)r.loop_launches,
                (double)r.feed_pieces, (double)r.device_peak_bytes};
  int m = (int)(sizeof(v) / sizeof(v[0]));
  for (int i = 0; i < n && i < m; i++) out[i] = v[i];
  return m;
}

void *yttm_api_open(const char *model_path, int n_threads) {
  Status st;
  auto *h = new Handle();
  h->enc = new BaseEncoder(std::string(model_path), n_threads, &st);
  if (!st.ok()) {
    g_err = st.message;
    delete h->enc;
    delete h;
    return nullptr;
  }
  return h;
}

void yttm_api_close(void *hv) {
  auto *h = static_cast<Handle *>(hv);
  if (!h) return;
  delete h->enc;
  delete h;
}

int yttm_api_vocab_size(void *hv) { return static_cast<Handle *>(hv)->enc->vocab_size(); }

void yttm_api_set_dropout_seed(void *hv, uint64_t seed) {
  auto *h = static_cast<Handle *>(hv);
  std::lock_guard<std::mutex> lock(h->mu);
  h->enc->set_dropout_seed(seed);
}

int yttm_api_encode_ids(void *hv, const char *bytes, const uint64_t *offsets, uint64_t n_sent, int bos, int eos,
                        int reverse, double dropout, uint64_t *total_ids) {
  auto *h = static_cast<Handle *>(hv);
  std::lock_guard<std::mutex> lock(h->mu);
  Status st = h->enc->encode_packed(bytes, offsets, n_sent, &g_res.ids, &g_res.offs, bos != 0, eos != 0, reverse != 0,
                                    dropout);
  if (!st.ok()) return fail(h, st.message);
  *total_ids = g_res.ids.size();
  return 0;
}

void yttm_api_result_ids(void *, int32_t *ids, uint64_t *offsets) {  // the calling thread's last encode_ids
  if (!g_res.ids.empty()) std::memcpy(ids, g_res.ids.data(), g_res.ids.size() * 4);
  std::memcpy(offsets, g_res.offs.data(), g_res.offs.size() * 8);
}

// One call, caller-supplied buffers (ids_cap >= bytes + 3 * n_sent always suffices).  Returns 0, 1 (error) or 2 (ids_cap
// too small: *total_ids holds the size needed, nothing written).
int yttm_api_encode_ids_into(void *hv, const char *bytes, const uint64_t *offsets, uint64_t n_sent, int bos, int eos,
                             int reverse, double dropout, int32_t *ids_out, uint64_t ids_cap, uint64_t *offsets_out,
                             uint64_t *total_ids) {
  auto *h = static_cast<Handle *>(hv);
  std::lock_guard<std::mutex> lock(h->mu);
  return ret(h, h->enc->encode_packed_into(bytes, offsets, n_sent, ids_out, ids_cap, offsets_out, total_ids, bos != 0, eos != 0,
                                           reverse != 0, dropout));
}

// Device-resident input and output (torch / CuPy callers): pointers into library-owned device memory, valid until the
// next encode call on this handle — callers that share a handle between threads copy the result out under their own lock.
int yttm_api_encode_device(void *hv, const char *d_bytes, const uint64_t *d_offsets, uint64_t n_bytes, uint64_t n_sent, int bos,
                           int eos, int reverse, double dropout, const int32_t **d_ids, const uint64_t **d_id_offsets,
                           uint64_t *total_ids) {
  auto *h = static_cast<Handle *>(hv);
  std::lock_guard<std::mutex> lock(h->mu);
  return ret(h, h->enc->encode_packed_device(d_bytes, d_offsets, n_bytes, n_sent, d_ids, d_id_offsets, total_ids, bos != 0,
                                             eos != 0, reverse != 0, dropout));
}

// Pieces come back length-framed (no in-band separator: a piece may hold any character, U+0001 included):
// yttm_api_result_counts -> (pieces, sentences), yttm_api_result_text -> the bytes, yttm_api_result_offsets -> byte
// offset of every piece (+ end) and first piece of every sentence (+ end).  Returns the byte length or -1.
int64_t yttm_api_encode_subwords(void *hv, const char *bytes, const uint64_t *offsets, uint64_t n_sent, int bos,
                                 int eos, int reverse, double dropout) {
  auto *h = static_cast<Handle *>(hv);
  std::vector<std::string> s(n_sent);
  for (uint64_t i = 0; i < n_sent; i++) s[i].assign(bytes + offsets[i], bytes + offsets[i + 1]);
  std::vector<std::vector<std::string>> out;
  {
    std::lock_guard<std::mutex> lock(h->mu);
    Status st = h->enc->encode_as_subwords(s, &out, bos != 0, eos != 0, reverse != 0, dropout);
    if (!st.ok()) { fail(h, st.message); return -1; }
  }
  g_res.clear_text();
  for (auto &sent : out) {
    for (auto &p : sent) g_res.add_piece(p);
    g_res.end_sentence();
  }
  return (int64_t)g_res.text.size();
}

// Spans and subwords on the GPU: caller-owned host buffers (return code 2: a capacity too small, sizes needed in the
// counts) or pointers into library-owned device memory valid until the next encode call on this handle.
int yttm_api_encode_spans_into(void *hv, const char *bytes, const uint64_t *offsets, uint64_t n_sent, int bos, int eos,
                               int reverse, double dropout, int32_t *ids_out, uint64_t ids_cap, uint64_t *offsets_out,
                               uint64_t *spans_out, uint64_t *total_ids) {
  auto *h = static_cast<Handle *>(hv);
  std::lock_guard<std::mutex> lock(h->mu);
  return ret(h, h->enc->encode_spans_into(bytes, offsets, n_sent, ids_out, ids_cap, offsets_out, spans_out, total_ids,
                                          bos != 0, eos != 0, reverse != 0, dropout));
}

int yttm_api_encode_spans_device(void *hv, const char *d_bytes, const uint64_t *d_offsets, uint64_t n_bytes, uint64_t n_sent,
                                 int bos, int eos, int reverse, double dropout, const int32_t **d_ids,
                                 const uint64_t **d_id_offsets, const uint64_t **d_spans, uint64_t *total_ids) {
  auto *h = static_cast<Handle *>(hv);
  std::lock_guard<std::mutex> lock(h->mu);
  return ret(h, h->enc->encode_spans_device(d_bytes, d_offsets, n_bytes, n_sent, d_ids, d_id_offsets, d_spans, total_ids,
                                            bos != 0, eos != 0, reverse != 0, dropout));
}

// Padded rows (yttm_enc_run_padded*): pad_id = YTTM_PAD_FROM_MODEL takes the model's pad id
int yttm_api_encode_padded_into(void *hv, const char *bytes, const uint64_t *offsets, uint64_t n_sent, int bos, int eos,
                                int reverse, double dropout, uint64_t width, int64_t pad_id, int32_t *ids_out,
                                uint64_t *lengths_out, uint64_t *spans_out) {
  auto *h = static_cast<Handle *>(hv);
  std::lock_guard<std::mutex> lock(h->mu);
  return ret(h, h->enc->encode_padded_into(bytes, offsets, n_sent, width, ids_out, lengths_out, spans_out, bos != 0, eos != 0,
                                           reverse != 0, dropout, pad_id));
}

int yttm_api_encode_padded_device(void *hv, const char *d_bytes, const uint64_t *d_offsets, uint64_t n_bytes, uint64_t n_sent,
                                  int bos, int eos, int reverse, double dropout, uint64_t width, int64_t pad_id, int with_spans,
                                  const int32_t **d_ids, const uint64_t **d_lengths, const uint64_t **d_spans,
                                  uint32_t *out_width) {
  auto *h = static_cast<Handle *>(hv);
  std::lock_guard<std::mutex> lock(h->mu);
  return ret(h, h->enc->encode_padded_device(d_bytes, d_offsets, n_bytes, n_sent, width, with_spans != 0, d_ids, d_lengths,
                                             d_spans, out_width, bos != 0, eos != 0, reverse != 0, dropout, pad_id));
}

// Overlapping windows (yttm_enc_run_windows_device): pad_id as for the padded rows
int yttm_api_encode_windows_device(void *hv, const char *d_bytes, const uint64_t *d_offsets, uint64_t n_bytes,
                                   uint64_t n_sent, int bos, int eos, int reverse, double dropout, uint64_t width,
                                   uint64_t stride, int64_t pad_id, int with_spans, const int32_t **d_ids,
                                   const uint64_t **d_lengths, const uint64_t **d_sentence, const uint64_t **d_start,
                                   const uint64_t **d_spans, uint64_t *n_rows) {
  auto *h = static_cast<Handle *>(hv);
  std::lock_guard<std::mutex> lock(h->mu);
  return ret(h, h->enc->encode_windows_device(d_bytes, d_offsets, n_bytes, n_sent, width, stride, with_spans != 0, d_ids,
                                              d_lengths, d_sentence, d_start, d_spans, n_rows, bos != 0, eos != 0,
                                              reverse != 0, dropout, pad_id));
}

int yttm_api_encode_subwords_into(void *hv, const char *bytes, const uint64_t *offsets, uint64_t n_sent, int bos, int eos,
                                  int reverse, double dropout, uint8_t *pieces, uint64_t bytes_cap, uint64_t *piece_offsets,
                                  uint64_t pieces_cap, uint64_t *sent_offsets, uint64_t *n_pieces, uint64_t *n_bytes) {
  auto *h = static_cast<Handle *>(hv);
  std::lock_guard<std::mutex> lock(h->mu);
  return ret(h, h->enc->encode_subwords_into(bytes, offsets, n_sent, pieces, bytes_cap, piece_offsets, pieces_cap, sent_offsets,
                                             n_pieces, n_bytes, bos != 0, eos != 0, reverse != 0, dropout));
}

int yttm_api_encode_subwords_device(void *hv, const char *d_bytes, const uint64_t *d_offsets, uint64_t n_bytes,
                                    uint64_t n_sent, int bos, int eos, int reverse, double dropout, const uint8_t **d_pieces,
                                    const uint64_t **d_piece_offsets, const uint64_t **d_sent_offsets, uint64_t *n_pieces,
                                    uint64_t *n_piece_bytes) {
  auto *h = static_cast<Handle *>(hv);
  std::lock_guard<std::mutex> lock(h->mu);
  return ret(h, h->enc->encode_subwords_device(d_bytes, d_offsets, n_bytes, n_sent, d_pieces, d_piece_offsets, d_sent_offsets,
                                               n_pieces, n_piece_bytes, bos != 0, eos != 0, reverse != 0, dropout));
}

void yttm_api_result_counts(void *, uint64_t *n_pieces, uint64_t *n_sentences) {
  *n_pieces = g_res.piece_off.size() - 1;
  *n_sentences = g_res.sent_off.size() - 1;
}
void yttm_api_result_text(void *, char *out) { std::memcpy(out, g_res.text.data(), g_res.text.size()); }
void yttm_api_result_offsets(void *, uint64_t *piece_off, uint64_t *sent_off) {
  std::memcpy(piece_off, g_res.piece_off.data(), g_res.piece_off.size() * 8);
  if (sent_off) std::memcpy(sent_off, g_res.sent_off.data(), g_res.sent_off.size() * 8);
}

int64_t yttm_api_decode(void *hv, const int32_t *ids, const uint64_t *offsets, uint64_t n_sent,
                        const int32_t *ignore, uint64_t n_ignore) {  // one piece per sentence
  auto *h = static_cast<Handle *>(hv);
  std::unordered_set<int> ign(ignore, ignore + n_ignore);
  g_res.clear_text();
  for (uint64_t i = 0; i < n_sent; i++) {
    std::vector<int> v(ids + offsets[i], ids + offsets[i + 1]);
    std::string sent;
    Status st = h->enc->decode(v, &sent, &ign);
    if (!st.ok()) { fail(h, st.message); return -1; }
    g_res.add_piece(sent);
    g_res.end_sentence();
  }
  return (int64_t)g_res.text.size();
}

// decode on the GPU into caller-supplied buffers: 0, 1 (error) or 2 (text_cap too small: *total_bytes holds the size
// needed, nothing written)
int yttm_api_decode_into(void *hv, const int32_t *ids, const uint64_t *offsets, uint64_t n_sent, const int32_t *ignore,
                         uint64_t n_ignore, uint8_t *text, uint64_t text_cap, uint64_t *text_offsets, uint64_t *total_bytes) {
  auto *h = static_cast<Handle *>(hv);
  std::lock_guard<std::mutex> lock(h->mu);
  return ret(h, h->enc->decode_packed_into(ids, offsets, n_sent, ignore, n_ignore, text, text_cap, text_offsets, total_bytes));
}

// decode of device-resident ids: pointers into library-owned device memory, valid until the next decode_device call on
// this handle (callers that share a handle between threads copy the result out under their own lock)
int yttm_api_decode_device(void *hv, const int32_t *d_ids, uint64_t n_ids, const uint64_t *d_offsets, uint64_t n_sent,
                           const int32_t *ignore, uint64_t n_ignore, const uint8_t **d_text, const uint64_t **d_text_offsets,
                           uint64_t *total_bytes) {
  auto *h = static_cast<Handle *>(hv);
  std::lock_guard<std::mutex> lock(h->mu);
  return ret(h, h->enc->decode_packed_device(d_ids, n_ids, d_offsets, n_sent, ignore, n_ignore, d_text, d_text_offsets,
                                             total_bytes));
}

int64_t yttm_api_id_to_subword(void *hv, int id) {
  auto *h = static_cast<Handle *>(hv);
  std::string piece;
  Status st = h->enc->id_to_subword(id, &piece);
  if (!st.ok()) { fail(h, st.message); return -1; }
  g_res.clear_text();
  g_res.add_piece(piece);
  g_res.end_sentence();
  return (int64_t)g_res.text.size();
}

int yttm_api_subword_to_id(void *hv, const char *subword) {
  return static_cast<Handle *>(hv)->enc->subword_to_id(subword);
}

int64_t yttm_api_vocab(void *hv) {  // length-framed like every piece list (yttm_api_result_counts / _offsets)
  auto *h = static_cast<Handle *>(hv);
  g_res.clear_text();
  for (auto &p : h->enc->vocabulary()) g_res.add_piece(p);
  g_res.end_sentence();
  return (int64_t)g_res.text.size();
}

int yttm_api_encode_cli(void *hv, const char *output_type, int stream, int bos, int eos, int reverse, double dropout) {
  auto *h = static_cast<Handle *>(hv);
  std::lock_guard<std::mutex> lock(h->mu);
  Status st = h->enc->encode_cli(output_type, stream != 0, bos != 0, eos != 0, reverse != 0, dropout);
  if (!st.ok()) return fail(h, st.message);
  return 0;
}
int yttm_api_encode_file(void *hv, int in_fd, const char *out_path, int text, int bos, int eos, int reverse,
                         double dropout, uint64_t *stats) {
  auto *h = static_cast<Handle *>(hv);
  std::lock_guard<std::mutex> lock(h->mu);
  return ret(h, h->enc->encode_file(in_fd, out_path, text != 0, bos != 0, eos != 0, reverse != 0, dropout, stats,
                                    stats + 1, stats + 2));
}
int yttm_api_encode_file_subwords(void *hv, int in_fd, const char *out_path, int bos, int eos, int reverse,
                                  double dropout, uint64_t *stats) {
  auto *h = static_cast<Handle *>(hv);
  std::lock_guard<std::mutex> lock(h->mu);
  return ret(h, h->enc->encode_file_subwords(in_fd, out_path, bos != 0, eos != 0, reverse != 0, dropout, stats,
                                             stats + 1, stats + 2));
}
int yttm_api_decode_file(void *hv, int in_fd, const char *in_prefix, const char *out_path, int text,
                         const int32_t *ignore, uint64_t n_ignore, uint64_t *stats) {
  auto *h = static_cast<Handle *>(hv);
  std::lock_guard<std::mutex> lock(h->mu);
  return ret(h, h->enc->decode_file(in_fd, in_prefix ? in_prefix : "", out_path, text != 0,
                                    std::vector<int32_t>(ignore, ignore + n_ignore), stats, stats + 1, stats + 2));
}
int yttm_api_decode_cli(void *hv, const int32_t *ignore, uint64_t n_ignore) {
  auto *h = static_cast<Handle *>(hv);
  std::unordered_set<int> ign(ignore, ignore + n_ignore);
  Status st = h->enc->decode_cli(&ign);
  if (!st.ok()) return fail(h, st.message);
  return 0;
}
void yttm_api_vocab_cli(void *hv, int verbose) { static_cast<Handle *>(hv)->enc->vocab_cli(verbose != 0); }

int yttm_api_dump_order(const uint32_t *filled, uint64_t n, uint32_t *out) {
  const std::vector<uint32_t> o = reference_dump_order(std::vector<uint32_t>(filled, filled + n));
  if (o.size() != n) return 1;  // duplicate keys in `filled`
  std::copy(o.begin(), o.end(), out);
  return 0;
}

int yttm_api_redump(const char *in_path, const char *out_path) {
  BPEState st;
  if (!st.load(in_path).ok()) return 1;
  st.dump(out_path);
  return 0;
}

// raw handles for bench.py / tests that drive the device ABI of yttm_b200.h directly
void *yttm_api_device_context(void *hv) { return static_cast<Handle *>(hv)->enc->device_context(); }
void *yttm_api_device_encoder(void *hv) { return static_cast<Handle *>(hv)->enc->device_encoder(); }

}  // extern "C"
