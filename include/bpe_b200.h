// bpe_b200.h — host C++ surface of the H100 BPE trainer / encoder.
//
// Mirrors the reference's C++ API (youtokentome/cpp/bpe.h:19 train_bpe, :22-82 BaseEncoder;
// value types of utils.h:11-86) — same names, argument meaning and error behaviour — so code and
// tests written against the reference read the same.  Bodies are new: both hot paths run on the
// GPU through the C ABI of yttm_b200.h; there is no CPU fallback (a missing device is a Status
// error).  The namespace is `vkcom` on purpose: a translation unit that includes this header
// instead of the reference's bpe.h compiles unchanged.
#pragma once
#include <cstdint>
#include <functional>
#include <iostream>
#include <string>
#include <unordered_map>
#include <unordered_set>
#include <vector>

struct yttm_ctx;
struct yttm_enc;

namespace vkcom {

// the reference vendors ska::flat_hash_map (third_party/flat_hash_map.h); only the interface of
// a hash map is part of the API, so the standard container is used here
template <class K, class V>
using flat_hash_map = std::unordered_map<K, V>;
template <class K>
using flat_hash_set = std::unordered_set<K>;

const uint32_t SPACE_TOKEN = 9601;  // U+2581, utils.h:9

const std::string UNK_TOKEN = "<UNK>";
const std::string PAD_TOKEN = "<PAD>";
const std::string BOS_TOKEN = "<BOS>";
const std::string EOS_TOKEN = "<EOS>";

enum OutputType { ID, SUBWORD };

struct BPE_Rule {  // x + y -> z
  uint32_t x{0}, y{0}, z{0};
  BPE_Rule() = default;
  BPE_Rule(uint32_t x_, uint32_t y_, uint32_t z_) : x(x_), y(y_), z(z_) {}
  bool operator==(const BPE_Rule &o) const { return x == o.x && y == o.y && z == o.z; }
};

struct SpecialTokens {
  int pad_id = -1, unk_id = -1, bos_id = -1, eos_id = -1;
  SpecialTokens() = default;
  SpecialTokens(int pad, int unk, int bos, int eos) : pad_id(pad), unk_id(unk), bos_id(bos), eos_id(eos) {}
  uint32_t max_id() const;
  bool taken_id(int id) const;
  uint64_t n_special_tokens() const;
};

struct BpeConfig {
  double character_coverage = 1;
  int n_threads = 0;  // kept for signature compatibility; the GPU path ignores it
  SpecialTokens special_tokens;
  BpeConfig() = default;
  BpeConfig(double coverage, int threads, const SpecialTokens &st)
      : character_coverage(coverage), n_threads(threads), special_tokens(st) {}
};

struct Status {
  int code{0};
  std::string message;
  Status() = default;
  Status(int c, std::string m) : code(c), message(std::move(m)) {}
  const std::string &error_message() const { return message; }
  bool ok() const { return code == 0; }
};

struct BPEState {  // the model (utils.h:66-74); text format of utils.cpp:50-91
  flat_hash_map<uint32_t, uint32_t> char2id;
  std::vector<BPE_Rule> rules;
  SpecialTokens special_tokens;
  void dump(const std::string &file_name);
  Status load(const std::string &file_name);
};

struct DecodeResult {
  std::vector<int> ids;
  std::vector<std::string> pieces;
};

struct EncodingConfig {
  bool bos, eos, reverse;
  double dropout_prob;
};

bool is_space(uint32_t ch);
std::string encode_utf8(const std::vector<uint32_t> &text);
std::vector<uint32_t> decode_utf8(const char *begin, const char *end);
std::vector<uint32_t> decode_utf8(const std::string &utf8_text);

// Timings / sizes of the last training run on this thread (milliseconds from CUDA events,
// wall seconds for host phases); purely informational.
struct TrainReport {
  uint64_t n_bytes = 0, data_len = 0, n_words = 0, n_unique = 0, n_tokens = 0, n_pairs = 0, n_merges = 0;
  double read_s = 0, h2d_ms = 0, char_hist_ms = 0, word_count_ms = 0, tokenise_ms = 0, pair_hist_ms = 0,
         merge_loop_ms = 0, total_s = 0;
  uint64_t launches = 0;
  uint64_t loop_launches = 0;   // launches of the merge loop (more than one: a compaction or a table rebuild ran)
  uint64_t feed_pieces = 0;     // pieces of a fed corpus (0: it was loaded whole)
  uint64_t device_peak_bytes = 0;   // largest sum of the training context's device buffers
};
const TrainReport &last_train_report();
// train_bpe keeps one training context (device buffers of the corpus, word table, packed words, pair table) per host
// thread between calls; this frees the calling thread's.
void release_training_cache();
// Training contexts currently cached by all host threads of the process (0 unless YTTM_TRAIN_KEEP_CACHE is set).
int training_cache_held();

// bpe.h:19 — reads input_path, trains on the GPU, writes the model file.
Status train_bpe(const std::string &input_path, const std::string &model_path, int vocab_size, BpeConfig config);

// learn_bpe_from_string (bpe.cpp:859; declared by the reference's tests in stress_test.h:8-13).
Status learn_bpe_from_string(std::string &text_utf8, int n_tokens, const std::string &output_file,
                             BpeConfig bpe_config, BPEState *bpe_state);

// compute_alphabet_helper (bpe.cpp:316-355) on a sparse histogram.
flat_hash_map<uint32_t, uint32_t> compute_alphabet_helper(const flat_hash_map<uint32_t, uint64_t> &char_cnt,
                                                          uint64_t data_len,
                                                          std::unordered_set<uint32_t> &removed_chars,
                                                          const BpeConfig &bpe_config);

// Order of the char2id lines in the reference's model file (BPEState::dump, utils.cpp:57-59, iterates a
// ska::flat_hash_map): `filled` = code points in the order the reference inserted them (U+2581, then by
// ascending id) -> the same code points in the order the reference's dump lists them.  Host only.
std::vector<uint32_t> reference_dump_order(const std::vector<uint32_t> &filled);

// Device selection for this process: YTTM_DEVICE env var, else LOCAL_RANK, else 0.
int default_device();

class BaseEncoder {
 public:
  BPEState bpe_state;
  flat_hash_map<uint32_t, uint32_t> id2char;
  flat_hash_map<uint32_t, std::vector<uint32_t>> recipe;
  flat_hash_map<std::string, uint32_t> reversed_recipe;
  flat_hash_map<uint64_t, int> rule2id;
  int n_threads;

  explicit BaseEncoder(BPEState bpe_state, int n_threads);
  explicit BaseEncoder(const std::string &model_path, int n_threads, Status *ret_status);
  ~BaseEncoder();
  BaseEncoder(const BaseEncoder &) = delete;
  BaseEncoder &operator=(const BaseEncoder &) = delete;

  void fill_from_state();

  Status encode_as_ids(const std::vector<std::string> &sentences, std::vector<std::vector<int>> *ids,
                       bool bos = false, bool eos = false, bool reverse = false, double dropout_prob = 0) const;
  Status encode_as_subwords(const std::vector<std::string> &sentences, std::vector<std::vector<std::string>> *subwords,
                            bool bos = false, bool eos = false, bool reverse = false, double dropout_prob = 0) const;

  // Additive zero-marshalling form of encode_as_ids: sentence i = bytes[offsets[i], offsets[i+1]).
  Status encode_packed(const char *bytes, const uint64_t *offsets, uint64_t n_sentences, std::vector<int32_t> *ids,
                       std::vector<uint64_t> *id_offsets, bool bos = false, bool eos = false, bool reverse = false,
                       double dropout_prob = 0) const;

  // The same into caller-owned buffers, one call: Status code 2 (nothing written, *total_ids = size needed) when
  // ids_cap is too small; ids_cap >= bytes + 3 * n_sentences always suffices.
  Status encode_packed_into(const char *bytes, const uint64_t *offsets, uint64_t n_sentences, int32_t *ids, uint64_t ids_cap,
                            uint64_t *id_offsets, uint64_t *total_ids, bool bos = false, bool eos = false,
                            bool reverse = false, double dropout_prob = 0) const;
  // DEVICE-resident input (d_bytes, d_offsets) and results left on the device: *d_ids / *d_id_offsets point into
  // library-owned memory that stays valid until the next encode call on this object.
  Status encode_packed_device(const char *d_bytes, const uint64_t *d_offsets, uint64_t n_bytes, uint64_t n_sentences,
                              const int32_t **d_ids, const uint64_t **d_id_offsets, uint64_t *total_ids, bool bos = false,
                              bool eos = false, bool reverse = false, double dropout_prob = 0) const;

  // encode_packed_into plus the source bytes of every id: spans[2j], spans[2j+1] = [start, end) of id j in the
  // coordinates of offsets (yttm_enc_run_spans in yttm_b200.h says which bytes an id covers).  spans holds
  // 2 * ids_cap values.  With dropout, advances the same sentence counter as encode_packed.
  Status encode_spans_into(const char *bytes, const uint64_t *offsets, uint64_t n_sentences, int32_t *ids, uint64_t ids_cap,
                           uint64_t *id_offsets, uint64_t *spans, uint64_t *total_ids, bool bos = false, bool eos = false,
                           bool reverse = false, double dropout_prob = 0) const;
  Status encode_spans_device(const char *d_bytes, const uint64_t *d_offsets, uint64_t n_bytes, uint64_t n_sentences,
                             const int32_t **d_ids, const uint64_t **d_id_offsets, const uint64_t **d_spans,
                             uint64_t *total_ids, bool bos = false, bool eos = false, bool reverse = false,
                             double dropout_prob = 0) const;
  // encode_packed as rows of an [n_sentences, width] matrix (yttm_enc_run_padded in yttm_b200.h gives the definition):
  // ids holds n_sentences * width cells, lengths n_sentences, spans (nullptr = not asked for) 2 * n_sentences * width.
  // width >= max(1, bos + eos).  pad_id = kModelPad takes the model's pad id (an error if the model has none).  With
  // dropout, advances the same sentence counter as encode_packed.
  static constexpr int64_t kModelPad = INT64_MIN;
  Status encode_padded_into(const char *bytes, const uint64_t *offsets, uint64_t n_sentences, uint64_t width, int32_t *ids,
                            uint64_t *lengths, uint64_t *spans, bool bos = false, bool eos = false, bool reverse = false,
                            double dropout_prob = 0, int64_t pad_id = kModelPad) const;
  // DEVICE-resident input; width = 0 takes the longest row, *out_width = the width used.  *d_ids / *d_lengths /
  // *d_spans (with_spans) point into library-owned memory that stays valid until the next encode call on this object.
  Status encode_padded_device(const char *d_bytes, const uint64_t *d_offsets, uint64_t n_bytes, uint64_t n_sentences,
                              uint64_t width, bool with_spans, const int32_t **d_ids, const uint64_t **d_lengths,
                              const uint64_t **d_spans, uint32_t *out_width, bool bos = false, bool eos = false,
                              bool reverse = false, double dropout_prob = 0, int64_t pad_id = kModelPad) const;
  // encode_as_subwords of a packed batch on the GPU, the pieces back to back: piece k = pieces[piece_offsets[k],
  // piece_offsets[k+1]), the pieces of sentence i = [sent_offsets[i], sent_offsets[i+1]).  Status code 2 (nothing
  // written, *n_pieces / *n_bytes = sizes needed) when pieces_cap (piece_offsets holds pieces_cap + 1) or bytes_cap
  // is too small.
  Status encode_subwords_into(const char *bytes, const uint64_t *offsets, uint64_t n_sentences, uint8_t *pieces,
                              uint64_t bytes_cap, uint64_t *piece_offsets, uint64_t pieces_cap, uint64_t *sent_offsets,
                              uint64_t *n_pieces, uint64_t *n_bytes, bool bos = false, bool eos = false, bool reverse = false,
                              double dropout_prob = 0) const;
  Status encode_subwords_device(const char *d_bytes, const uint64_t *d_offsets, uint64_t n_bytes, uint64_t n_sentences,
                                const uint8_t **d_pieces, const uint64_t **d_piece_offsets, const uint64_t **d_sent_offsets,
                                uint64_t *n_pieces, uint64_t *n_piece_bytes, bool bos = false, bool eos = false,
                                bool reverse = false, double dropout_prob = 0) const;

  // decode() of a packed batch on the GPU: sentence i = ids[offsets[i], offsets[i+1]), text i =
  // text[text_offsets[i], text_offsets[i+1]).  Status code 2 (nothing written, *total_bytes = size needed) when
  // text_cap is too small.
  Status decode_packed_into(const int32_t *ids, const uint64_t *offsets, uint64_t n_sentences, const int32_t *ignore_ids,
                            uint64_t n_ignore, uint8_t *text, uint64_t text_cap, uint64_t *text_offsets,
                            uint64_t *total_bytes) const;
  // DEVICE-resident ids[n_ids] / offsets, results left on the device: *d_text / *d_text_offsets point into
  // library-owned memory that stays valid until the next decode_packed_device call on this object.
  Status decode_packed_device(const int32_t *d_ids, uint64_t n_ids, const uint64_t *d_offsets, uint64_t n_sentences,
                              const int32_t *ignore_ids, uint64_t n_ignore, const uint8_t **d_text,
                              const uint64_t **d_text_offsets, uint64_t *total_bytes) const;

  Status id_to_subword(int id, std::string *subword, bool replace_space = false) const;
  int subword_to_id(const std::string &token) const;

  Status decode(const std::vector<std::vector<int>> &ids, std::vector<std::string> *sentences,
                const std::unordered_set<int> *ignore_ids) const;
  Status decode(const std::vector<int> &ids, std::string *sentence, const std::unordered_set<int> *ignore_ids) const;
  Status decode(const std::vector<std::string> &ids, std::vector<std::string> *sentences,
                const std::unordered_set<int> *ignore_ids) const;

  int vocab_size() const;
  std::vector<std::string> vocabulary() const;

  Status encode_cli(const std::string &output_type, bool stream, bool bos = false, bool eos = false,
                    bool reverse = false, double dropout_prob = 0) const;
  Status decode_cli(const std::unordered_set<int> *ignore_ids) const;
  void vocab_cli(bool verbose) const;

  // BPE-dropout stream: seed of the counter-based generator and the running sentence counter
  // (replaces the reference's global std::mt19937, bpe.cpp:1415).
  void set_dropout_seed(uint64_t seed) const { dropout_seed_ = seed; sentence_counter_ = 0; }

  yttm_ctx *device_context() const { return ctx_; }
  yttm_enc *device_encoder() const { return enc_; }

 private:
  Status init_device();
  Status resolve_pad(int64_t pad_id, int32_t *out) const;  // encode_padded_*: kModelPad -> the model's pad id
  // The frame of every encode_*_into / _device and decode_packed_* call: the <BOS> / <EOS> check, `checked` (an argument
  // error the caller found), the device status, then call() (a yttm_enc_run* / yttm_dec_run* call): its return code 2 is
  // Status 2 ("<name>: output buffer too small"), any other error the context's message.  With dropout, a call that
  // succeeds advances the sentence counter by n_sent.
  Status run_device(const char *name, bool bos, bool eos, double dropout_prob, uint64_t n_sent,
                    const std::function<int()> &call, const Status &checked = Status()) const;
  mutable yttm_ctx *ctx_ = nullptr;
  mutable yttm_enc *enc_ = nullptr;
  mutable uint64_t dropout_seed_ = 5489;  // std::mt19937's default seed, for flavour
  mutable uint64_t sentence_counter_ = 0;
  Status device_status_;
};

}  // namespace vkcom
