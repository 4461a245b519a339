// bpe_host.cpp — host C++ above the C ABI: train_bpe / BaseEncoder with the reference's surface
// (youtokentome/cpp/bpe.h) and model file format (utils.cpp:50-91).  Everything data-parallel
// goes through include/yttm_b200.h to the GPU; what stays here is O(alphabet + vocab) glue:
// config validation, the coverage cut (the only floating point of training), id renaming,
// model I/O, id <-> subword tables, decode.
#include <algorithm>
#include <atomic>
#include <cassert>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <functional>
#include <sstream>
#include <thread>

#include "../../include/bpe_b200.h"
#include "../../include/yttm_b200.h"
#include "common.cuh"

namespace vkcom {

namespace {
double now_s() { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); }
thread_local TrainReport g_report;
std::string ctx_err(yttm_ctx *c) { return std::string(yttm_last_error(c)); }
}  // namespace

const TrainReport &last_train_report() { return g_report; }

// ---------------------------------------------------------------------------------------------
// small value types (utils.cpp:19-44)
// ---------------------------------------------------------------------------------------------
uint32_t SpecialTokens::max_id() const { return (uint32_t)std::max({0, unk_id, pad_id, bos_id, eos_id}); }
bool SpecialTokens::taken_id(int id) const { return id == unk_id || id == pad_id || id == bos_id || id == eos_id; }
uint64_t SpecialTokens::n_special_tokens() const {
  return (uint64_t)(unk_id != -1) + (pad_id != -1) + (bos_id != -1) + (eos_id != -1);
}

bool is_space(uint32_t ch) { return ch == 32 || (ch >= 9 && ch <= 13) || ch == SPACE_TOKEN; }  // utils.cpp:99-101

// ---------------------------------------------------------------------------------------------
// host UTF-8 (utf8.cpp:76-132) — only used for pieces / decode / vocab, never on the hot path
// ---------------------------------------------------------------------------------------------
static void append_utf8(uint32_t x, std::string *out) {
  if (x <= 0x7f) out->push_back((char)x);
  else if (x <= 0x7ff) { out->push_back((char)(0xc0 | (x >> 6))); out->push_back((char)(0x80 | (x & 0x3f))); }
  else if (x <= 0xffff) {
    out->push_back((char)(0xe0 | (x >> 12))); out->push_back((char)(0x80 | ((x >> 6) & 0x3f)));
    out->push_back((char)(0x80 | (x & 0x3f)));
  } else {
    out->push_back((char)(0xf0 | (x >> 18))); out->push_back((char)(0x80 | ((x >> 12) & 0x3f)));
    out->push_back((char)(0x80 | ((x >> 6) & 0x3f))); out->push_back((char)(0x80 | (x & 0x3f)));
  }
}
std::string encode_utf8(const std::vector<uint32_t> &text) {
  std::string s;
  for (uint32_t c : text) append_utf8(c, &s);
  return s;
}
static const uint32_t INVALID_UNICODE = 0x0fffffff;
static uint32_t decode_one(const unsigned char *p, size_t size, size_t *len) {
  auto cont = [](unsigned char b) { return (b & 0xc0) == 0x80; };
  auto okcp = [](uint32_t x) { return x < 0xd800 || (x > 0xdfff && x < 0x110000); };
  unsigned char b0 = p[0];
  *len = 1;
  if (b0 < 0x80) return b0;
  if ((b0 & 0xe0) == 0xc0 && size >= 2 && cont(p[1])) {
    uint32_t cp = ((b0 & 0x1fu) << 6) | (p[1] & 0x3fu);
    if (cp >= 0x80 && okcp(cp)) { *len = 2; return cp; }
  } else if ((b0 & 0xf0) == 0xe0 && size >= 3 && cont(p[1]) && cont(p[2])) {
    uint32_t cp = ((b0 & 0x0fu) << 12) | ((p[1] & 0x3fu) << 6) | (p[2] & 0x3fu);
    if (cp >= 0x800 && okcp(cp)) { *len = 3; return cp; }
  } else if ((b0 & 0xf8) == 0xf0 && size >= 4 && cont(p[1]) && cont(p[2]) && cont(p[3])) {
    uint32_t cp = ((b0 & 0x07u) << 18) | ((p[1] & 0x3fu) << 12) | ((p[2] & 0x3fu) << 6) | (p[3] & 0x3fu);
    if (cp >= 0x10000 && okcp(cp)) { *len = 4; return cp; }
  }
  return INVALID_UNICODE;
}
std::vector<uint32_t> decode_utf8(const char *begin, const char *end) {
  std::vector<uint32_t> out;
  bool invalid = false;
  const unsigned char *p = (const unsigned char *)begin, *e = (const unsigned char *)end;
  while (p < e) {
    size_t len;
    uint32_t cp = decode_one(p, (size_t)(e - p), &len);
    if (cp != INVALID_UNICODE) out.push_back(cp); else invalid = true;
    p += len;
  }
  if (invalid) std::cerr << "WARNING Input contains invalid unicode characters." << std::endl;
  return out;
}
std::vector<uint32_t> decode_utf8(const std::string &s) { return decode_utf8(s.data(), s.data() + s.size()); }

// ---------------------------------------------------------------------------------------------
// model file (utils.cpp:50-91).  The reference writes the char2id lines in the iteration order of
// its ska::flat_hash_map (third_party/flat_hash_map.h), i.e. in the slot order of an
// open-addressing robin-hood table.  To make the dump byte-identical we replay, keys only, what
// happens to that table: compute_alphabet_helper inserts U+2581 and then the kept characters by
// descending (count, code point) (bpe.cpp:340-353) = ascending id, and `*bpe_state = {char2id,...}`
// (bpe.cpp:1289) copy-constructs it (flat_hash_map.h:361-375: size the new table for the other
// one, then re-insert in the other one's slot order).  Behaviour restated from the header:
//   * home slot of key k = (11400714819323198485 * k) >> shift, shift = 64 - log2(buckets)
//     (fibonacci_hash_policy :1274-1301; std::hash<uint32_t> is the identity);
//   * a table of b buckets has b + max_lookups slots, max_lookups = max(4, log2 b) (:803-807);
//   * emplace walks from the home slot while the resident is at least as far from its own home
//     (:578-593), then takes an empty slot or swaps with the "richer" resident and carries that
//     one on (:830-873); the table doubles (min 4 buckets) when it has none, when a walk reaches
//     max_lookups or when size + 1 > buckets / 2, re-inserting the old slots in ascending slot
//     order (:630-662, :875-878).
// ---------------------------------------------------------------------------------------------
namespace {
class SlotOrderReplay {
 public:
  void insert(uint32_t k) {
    for (;;) {
      if (buckets_ == 0) { rehash(4); continue; }
      uint64_t p = (11400714819323198485ull * (uint64_t)k) >> shift_;
      int d = 0;
      bool found = false;
      for (; dist_[p] >= d; ++p, ++d)
        if (key_[p] == k && p + 1 < dist_.size()) { found = true; break; }
      if (found) return;
      if (d == max_lookups_ || (double)(size_ + 1) > (double)buckets_ * 0.5) { rehash(2 * buckets_); continue; }
      if (dist_[p] < 0) { put(p, d, k); return; }
      // robin hood: the new key takes this slot, the displaced resident is carried forward
      const uint64_t taken = p;
      uint32_t carry = k;
      swap_in(p, d, carry);
      bool regrow = false;
      for (++d, ++p;; ++p) {
        if (dist_[p] < 0) { put(p, d, carry); return; }
        if (dist_[p] < d) { swap_in(p, d, carry); ++d; continue; }
        if (++d == max_lookups_) { regrow = true; break; }
      }
      if (regrow) {  // the carried resident goes back into the taken slot, the new key is retried after growing
        std::swap(carry, key_[taken]);
        rehash(2 * buckets_);
        k = carry;
      }
    }
  }
  // copy construction: rehash_for_other_container (:813-816) + insert(other.begin(), other.end())
  SlotOrderReplay copy() const {
    SlotOrderReplay c;
    c.rehash(std::min<uint64_t>(2 * size_, buckets_));
    for (uint32_t k : order()) c.insert(k);
    return c;
  }
  std::vector<uint32_t> order() const {
    std::vector<uint32_t> out;
    for (size_t i = 0; i + 1 < dist_.size(); i++)
      if (dist_[i] >= 0) out.push_back(key_[i]);
    return out;
  }

 private:
  void put(uint64_t p, int d, uint32_t k) { dist_[p] = (int8_t)d; key_[p] = k; ++size_; }
  void swap_in(uint64_t p, int &d, uint32_t &k) {
    const int od = dist_[p];
    dist_[p] = (int8_t)d;
    d = od;
    std::swap(k, key_[p]);
  }
  static int log2u(uint64_t v) { int r = 0; while (v >>= 1) ++r; return r; }
  void rehash(uint64_t want) {
    want = std::max<uint64_t>(want, (uint64_t)std::ceil((double)size_ / 0.5));
    if (want == 0) return;  // nothing allocated yet and nothing to hold
    uint64_t b = 2;
    while (b < want) b <<= 1;
    if (b == buckets_) return;
    const std::vector<uint32_t> old = order();
    buckets_ = b;
    shift_ = 64 - log2u(b);
    max_lookups_ = std::max(4, log2u(b));
    dist_.assign(b + max_lookups_, (int8_t)-1);
    key_.assign(b + max_lookups_, 0u);
    dist_.back() = 0;  // the end marker is "occupied at distance 0" for the walks
    size_ = 0;
    for (uint32_t k : old) insert(k);
  }
  std::vector<int8_t> dist_;
  std::vector<uint32_t> key_;
  uint64_t buckets_ = 0, size_ = 0;
  int shift_ = 63, max_lookups_ = 3;
};
}  // namespace

// keys in the order the reference's char2id was filled -> keys in the order its dump lists them
std::vector<uint32_t> reference_dump_order(const std::vector<uint32_t> &insertion_order) {
  SlotOrderReplay t;
  for (uint32_t k : insertion_order) t.insert(k);
  return t.copy().order();
}

void BPEState::dump(const std::string &file_name) {
  std::ofstream fout(file_name, std::ios::out);
  if (fout.fail()) { std::cerr << "Can't open file: " << file_name << std::endl; assert(false); }
  fout << char2id.size() << " " << rules.size() << std::endl;
  std::vector<std::pair<uint32_t, uint32_t>> by_id;  // (id, code point): ids ascend in insertion order
  for (auto &kv : char2id) by_id.emplace_back(kv.second, kv.first);
  std::sort(by_id.begin(), by_id.end());
  std::vector<uint32_t> filled;
  for (auto &s : by_id) filled.push_back(s.second);
  for (uint32_t cp : reference_dump_order(filled)) fout << cp << " " << char2id.at(cp) << std::endl;
  for (auto &r : rules) fout << r.x << " " << r.y << " " << r.z << std::endl;
  fout << special_tokens.unk_id << " " << special_tokens.pad_id << " " << special_tokens.bos_id << " "
       << special_tokens.eos_id << std::endl;
}

Status BPEState::load(const std::string &file_name) {
  char2id.clear();
  rules.clear();
  std::ifstream fin(file_name, std::ios::in);
  if (fin.fail()) return Status(1, "Can not open file with model: " + file_name);
  int n, m;
  fin >> n >> m;
  for (int i = 0; i < n; i++) { uint32_t a, b; fin >> a >> b; char2id[a] = b; }
  for (int i = 0; i < m; i++) { uint32_t x, y, z; fin >> x >> y >> z; rules.emplace_back(x, y, z); }
  fin >> special_tokens.unk_id >> special_tokens.pad_id >> special_tokens.bos_id >> special_tokens.eos_id;
  return Status();
}

// ---------------------------------------------------------------------------------------------
// training
// ---------------------------------------------------------------------------------------------
int default_device() {
  if (const char *e = std::getenv("YTTM_DEVICE")) return std::atoi(e);
  if (const char *e = std::getenv("LOCAL_RANK")) return std::atoi(e);
  return 0;
}

// compute_alphabet_helper (bpe.cpp:316-355): sort (count, cp) ascending, drop the rarest while
// the remaining mass still exceeds data_len * coverage (compared in double, as the reference
// does), ids: [0, n_special) unused, U+2581, then kept chars by descending (count, cp).
flat_hash_map<uint32_t, uint32_t> compute_alphabet_helper(const flat_hash_map<uint32_t, uint64_t> &char_cnt,
                                                          uint64_t data_len,
                                                          std::unordered_set<uint32_t> &removed_chars,
                                                          const BpeConfig &bpe_config) {
  std::vector<std::pair<uint64_t, uint32_t>> freq;
  freq.reserve(char_cnt.size());
  for (auto &x : char_cnt) freq.emplace_back(x.second, x.first);
  std::sort(freq.begin(), freq.end());
  uint64_t cur = 0, n_removed = 0;
  for (; cur < freq.size() &&
         (double)(data_len - n_removed - freq[cur].first) > (double)data_len * bpe_config.character_coverage;
       cur++)
    n_removed += freq[cur].first;
  std::cerr << "number of unique characters in the training data: " << freq.size() << std::endl;
  std::cerr << "number of deleted characters: " << cur << std::endl;
  std::cerr << "number of unique characters left: " << freq.size() - cur << std::endl;
  flat_hash_map<uint32_t, uint32_t> char2id;
  uint64_t used_ids = bpe_config.special_tokens.n_special_tokens();
  char2id[SPACE_TOKEN] = (uint32_t)used_ids++;
  for (uint64_t i = 0; i < cur; i++) removed_chars.insert(freq[i].second);
  for (int64_t i = (int64_t)freq.size() - 1; i >= (int64_t)cur; i--)
    if (!is_space(freq[i].second)) char2id[freq[i].second] = (uint32_t)used_ids++;
  return char2id;
}

// check_config (bpe.cpp:1295-1350)
static Status check_config(BpeConfig &cfg, int vocab_size) {
  const SpecialTokens &st = cfg.special_tokens;
  if (cfg.character_coverage <= 0 || cfg.character_coverage > 1)
    return Status(1, "coverage value must be in the range (0, 1]. Current value of coverage = " +
                         std::to_string(cfg.character_coverage));
  if (st.unk_id < 0 || st.unk_id >= vocab_size)
    return Status(1, "unk_id: must be in the range [0, vocab_size - 1]. Current value of vocab_size = " +
                         std::to_string(vocab_size) + "; unk_id = " + std::to_string(st.unk_id));
  if (st.pad_id < -1 || st.pad_id >= vocab_size)
    return Status(1, "pad_id must be in the range [-1, vocab_size - 1]. Current value of vocab_size = " +
                         std::to_string(vocab_size) + "; pad_id = " + std::to_string(st.pad_id));
  if (st.bos_id < -1 || st.bos_id >= vocab_size)
    return Status(1, "bos_id must be in the range [-1, vocab_size - 1]. Current value of vocab_size = " +
                         std::to_string(vocab_size) + "; bos_id = " + std::to_string(st.bos_id));
  if (st.eos_id < -1 || st.eos_id >= vocab_size)
    return Status(1, "eos_id must be in the range [-1, vocab_size - 1]. Current value of vocab_size = " +
                         std::to_string(vocab_size) + " eos_id = " + std::to_string(st.eos_id));
  std::unordered_set<int> ids;
  uint64_t cnt = 0;
  if (st.pad_id != -1) { ids.insert(st.pad_id); cnt++; }
  if (st.bos_id != -1) { ids.insert(st.bos_id); cnt++; }
  if (st.eos_id != -1) { ids.insert(st.eos_id); cnt++; }
  ids.insert(st.unk_id); cnt++;
  if (ids.size() != cnt) return Status(1, "All ids of special tokens must be different.");
  if (cfg.n_threads == -1) cfg.n_threads = (int)std::thread::hardware_concurrency();
  cfg.n_threads = std::min(8, std::max(1, cfg.n_threads));
  return Status();
}

static void print_config(const std::string &in, const std::string &model, int vocab_size, const BpeConfig &c) {
  std::cerr << "Training parameters" << std::endl;
  std::cerr << "  input: " << in << std::endl;
  std::cerr << "  model: " << model << std::endl;
  std::cerr << "  vocab_size: " << vocab_size << std::endl;
  std::cerr << "  device: cuda:" << default_device() << " (n_threads=" << c.n_threads << " ignored)" << std::endl;
  std::cerr << "  character_coverage: " << c.character_coverage << std::endl;
  std::cerr << "  pad: " << c.special_tokens.pad_id << std::endl;
  std::cerr << "  unk: " << c.special_tokens.unk_id << std::endl;
  std::cerr << "  bos: " << c.special_tokens.bos_id << std::endl;
  std::cerr << "  eos: " << c.special_tokens.eos_id << std::endl;
  std::cerr << std::endl;
}

// rename_tokens (bpe.cpp:814-837): k-th internal id after the specials -> k-th free final id.
static void rename_tokens(flat_hash_map<uint32_t, uint32_t> &char2id, std::vector<BPE_Rule> &rules,
                          const SpecialTokens &st, uint32_t n_tokens) {
  std::vector<uint32_t> ren((size_t)n_tokens + st.n_special_tokens() + 1, 0);
  uint32_t cur = (uint32_t)st.n_special_tokens();
  for (uint32_t i = 0; i < n_tokens; i++)
    if (!st.taken_id((int)i)) ren[cur++] = i;
  for (auto &kv : char2id) kv.second = ren[kv.second];
  for (auto &r : rules) { r.x = ren[r.x]; r.y = ren[r.y]; r.z = ren[r.z]; }
}

struct TrainCache {  // deliberately not destroyed at thread / process exit (no CUDA calls during teardown)
  yttm_ctx *ctx = nullptr;
  int device = -1;
  std::string geometry;
};
static thread_local TrainCache g_train_cache;
static std::atomic<int> g_train_contexts_held{0};   // cached training contexts of all threads

static void drop_cached_context(TrainCache &cache) {
  if (!cache.ctx) return;
  yttm_ctx_destroy(cache.ctx);
  cache.ctx = nullptr;
  g_train_contexts_held--;
}

// Gives the device memory of this thread's cached training context back (the next train_bpe builds a new one).
void release_training_cache() {
  drop_cached_context(g_train_cache);
  g_train_cache.device = -1;
}

int training_cache_held() { return g_train_contexts_held.load(); }

// Gives a training context the corpus: yttm_train_load_corpus of one buffer, or yttm_train_feed_begin / feed / feed_end
// of blocks.  Returns the error text, empty on success.
using Ingest = std::function<std::string(yttm_ctx *)>;

static Status train_on_ctx(const Ingest &ingest, int n_tokens, const std::string &output_file, BpeConfig cfg,
                           BPEState *out_state) {
  double t_start = now_s();
  // The context holds the corpus, the word table, the packed words and the pair table (more than the corpus itself).
  // The reference's train_bpe is stateless, so the device memory goes back on every return, errors included;
  // YTTM_TRAIN_KEEP_CACHE=1 keeps the context for the next training of this thread (benchmarks, test loops),
  // release_training_cache() frees it.
  struct ReleaseUnlessKept {
    ~ReleaseUnlessKept() { if (!std::getenv("YTTM_TRAIN_KEEP_CACHE")) release_training_cache(); }
  } release_on_return;
  // one training context per host thread and device; with YTTM_TRAIN_KEEP_CACHE=1 it survives the call and its device
  // buffers (corpus, word table, packed words, pair table) are reused by the next training of this thread
  TrainCache &cache = g_train_cache;
  // a context fixes its launch geometry when it first trains: the knobs that shape it are part of the cache key, so a
  // changed setting takes effect in a running process (the A/B tools and the tests vary them between calls)
  std::string geometry;
  for (const char *const *k = yttm_geometry_knobs; *k; k++) {
    const char *v = std::getenv(*k);
    geometry += v ? v : "";
    geometry += '|';
  }
  if (cache.ctx && (cache.device != default_device() || cache.geometry != geometry)) drop_cached_context(cache);
  if (!cache.ctx) {
    if (yttm_ctx_create(default_device(), &cache.ctx)) { cache.ctx = nullptr; return Status(1, yttm_last_error(nullptr)); }
    g_train_contexts_held++;
    cache.device = default_device();
    cache.geometry = geometry;
  }
  yttm_ctx *ctx = cache.ctx;
  const uint64_t launches0 = yttm_launch_count(ctx);

  {
    std::string err = ingest(ctx);
    if (!err.empty()) return Status(1, err);
  }
  uint64_t data_len = 0, n_distinct = 0;
  if (yttm_train_char_hist(ctx, &data_len, &n_distinct)) return Status(1, ctx_err(ctx));
  std::vector<uint32_t> cps(n_distinct);
  std::vector<uint64_t> cnts(n_distinct);
  if (n_distinct) yttm_train_get_char_hist(ctx, cps.data(), cnts.data());
  flat_hash_map<uint32_t, uint64_t> char_cnt;
  for (uint64_t i = 0; i < n_distinct; i++) char_cnt[cps[i]] = cnts[i];
  std::unordered_set<uint32_t> removed;
  flat_hash_map<uint32_t, uint32_t> char2id = compute_alphabet_helper(char_cnt, data_len, removed, cfg);

  uint64_t used_ids = char2id.size() + cfg.special_tokens.n_special_tokens();
  if (used_ids > (uint64_t)n_tokens)  // bpe.cpp:1051-1062
    return Status(1, "Incorrect arguments. Vocabulary size too small. Set vocab_size>=" + std::to_string(used_ids) +
                         ".  Current value for vocab_size=" + std::to_string(n_tokens));

  std::vector<uint32_t> kcp, kid;
  for (auto &kv : char2id) { kcp.push_back(kv.first); kid.push_back(kv.second); }
  if (yttm_train_set_alphabet(ctx, kcp.data(), kid.data(), kcp.size(), char2id[SPACE_TOKEN]))
    return Status(1, ctx_err(ctx));
  yttm_train_stats st{};
  if (yttm_train_build(ctx, &st)) return Status(1, ctx_err(ctx));

  uint32_t max_merges = (uint32_t)((uint64_t)n_tokens - used_ids), n_done = 0;
  std::vector<uint32_t> xyz((size_t)max_merges * 3 + 3);
  std::vector<uint64_t> rf((size_t)max_merges + 1);
  if (yttm_train_run(ctx, (uint32_t)used_ids, max_merges, xyz.data(), rf.data(), &n_done))
    return Status(1, ctx_err(ctx));
  if (n_done < max_merges)
    std::cerr << "WARNING merged only: " << used_ids + n_done << " pairs of tokens" << std::endl;

  std::vector<BPE_Rule> rules;
  rules.reserve(n_done);
  for (uint32_t i = 0; i < n_done; i++) rules.emplace_back(xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2]);
  rename_tokens(char2id, rules, cfg.special_tokens, (uint32_t)n_tokens);

  BPEState state;
  state.char2id = char2id;
  state.rules = rules;
  state.special_tokens = cfg.special_tokens;
  if (!output_file.empty()) {
    std::ofstream probe(output_file, std::ios::out);
    if (probe.fail()) return Status(1, "Can't open file: " + output_file);
    probe.close();
    state.dump(output_file);
    std::cerr << "model saved to: " << output_file << std::endl;
  }
  if (out_state) *out_state = state;

  TrainReport &r = g_report;
  r.n_bytes = st.n_bytes; r.data_len = data_len; r.n_words = st.n_words; r.n_unique = st.n_unique; r.n_tokens = st.n_tokens;
  r.n_pairs = st.n_pairs; r.n_merges = n_done;
  r.h2d_ms = yttm_stage_ms(ctx, "h2d"); r.char_hist_ms = yttm_stage_ms(ctx, "char_hist");
  r.word_count_ms = yttm_stage_ms(ctx, "word_count"); r.tokenise_ms = yttm_stage_ms(ctx, "tokenise");
  r.pair_hist_ms = yttm_stage_ms(ctx, "pair_hist"); r.merge_loop_ms = yttm_stage_ms(ctx, "merge_loop");
  r.launches = yttm_launch_count(ctx) - launches0;
  r.loop_launches = (uint64_t)yttm_stage_ms(ctx, "loop_launches");
  r.feed_pieces = (uint64_t)yttm_stage_ms(ctx, "feed_pieces");
  r.device_peak_bytes = (uint64_t)yttm_stage_ms(ctx, "dev_peak_bytes");
  r.total_s = now_s() - t_start;
  return Status();
}

// Blocks of the corpus for a fed training: the host never needs more than one block, the device never the corpus.
constexpr uint64_t FEED_BLOCK = 16ull << 20;

static Status train_on_buffer(const char *text, uint64_t n, int n_tokens, const std::string &output_file,
                              BpeConfig cfg, BPEState *out_state) {
  return train_on_ctx([&](yttm_ctx *ctx) -> std::string {
    if (!yttm_train_feed_selected(ctx, n)) return yttm_train_load_corpus(ctx, text, n, 0) ? ctx_err(ctx) : "";
    if (yttm_train_feed_begin(ctx)) return ctx_err(ctx);
    for (uint64_t at = 0; at < n; at += FEED_BLOCK)
      if (yttm_train_feed(ctx, text + at, std::min(FEED_BLOCK, n - at))) return ctx_err(ctx);
    return yttm_train_feed_end(ctx, nullptr, nullptr) ? ctx_err(ctx) : "";
  }, n_tokens, output_file, cfg, out_state);
}

Status learn_bpe_from_string(std::string &text_utf8, int n_tokens, const std::string &output_file,
                             BpeConfig bpe_config, BPEState *bpe_state) {
  g_report = TrainReport();
  return train_on_buffer(text_utf8.data(), text_utf8.size(), n_tokens, output_file, bpe_config, bpe_state);
}

Status train_bpe(const std::string &input_path, const std::string &model_path, int vocab_size, BpeConfig cfg) {
  Status status = check_config(cfg, vocab_size);
  if (!status.ok()) return status;
  print_config(input_path, model_path, vocab_size, cfg);
  std::cerr << "reading file..." << std::endl;
  FILE *fin = std::fopen(input_path.c_str(), "rb");  // fast_read_file_utf8 (bpe.cpp:67-84)
  if (!fin) return Status(1, "Failed to open file: " + input_path);
  struct Closer { FILE *f; ~Closer() { std::fclose(f); } } closer{fin};
  // a file of known size is read whole and loaded, unless it is large enough to be fed (yttm_train_feed_selected); a
  // pipe or FIFO has no size and is always fed.  read_s: the host time spent blocked in reads.
  std::fseek(fin, 0, SEEK_END);
  long sz = std::ftell(fin);
  std::fseek(fin, 0, SEEK_SET);
  const uint64_t size = sz > 0 ? (uint64_t)sz : UINT64_MAX;
  double read_s = 0;
  std::string data;
  g_report = TrainReport();
  BPEState state;
  status = train_on_ctx([&](yttm_ctx *ctx) -> std::string {
    if (!yttm_train_feed_selected(ctx, size)) {
      double t0 = now_s();
      data.resize((size_t)size);
      data.resize(std::fread(&data[0], 1, (size_t)size, fin));
      read_s = now_s() - t0;
      std::cerr << "learning bpe..." << std::endl;
      return yttm_train_load_corpus(ctx, data.data(), data.size(), 0) ? ctx_err(ctx) : "";
    }
    std::cerr << "learning bpe (the corpus is fed in pieces)..." << std::endl;
    if (yttm_train_feed_begin(ctx)) return ctx_err(ctx);
    std::vector<char> block(FEED_BLOCK);
    for (;;) {
      double t0 = now_s();
      size_t got = std::fread(block.data(), 1, block.size(), fin);
      read_s += now_s() - t0;
      if (!got) break;
      if (yttm_train_feed(ctx, block.data(), got)) return ctx_err(ctx);
    }
    if (std::ferror(fin)) return "Failed to read file: " + input_path;
    return yttm_train_feed_end(ctx, nullptr, nullptr) ? ctx_err(ctx) : "";
  }, vocab_size, model_path, cfg, &state);
  g_report.read_s = read_s;
  return status;
}

// ---------------------------------------------------------------------------------------------
// encoder
// ---------------------------------------------------------------------------------------------
static std::string token2word(const std::vector<uint32_t> &source, const flat_hash_map<uint32_t, uint32_t> &id2char) {
  std::vector<uint32_t> res;
  res.reserve(source.size());
  for (uint32_t i : source) res.push_back(id2char.at(i));
  return encode_utf8(res);
}

BaseEncoder::BaseEncoder(BPEState state, int threads) : bpe_state(std::move(state)), n_threads(threads) {
  fill_from_state();
  if (n_threads == -1) n_threads = std::max(1, (int)std::thread::hardware_concurrency());
  device_status_ = init_device();
}

BaseEncoder::BaseEncoder(const std::string &model_path, int threads, Status *ret_status) : n_threads(threads) {
  Status status = bpe_state.load(model_path);
  if (!status.ok()) { *ret_status = status; return; }
  fill_from_state();
  if (n_threads == -1) n_threads = std::max(1, (int)std::thread::hardware_concurrency());
  device_status_ = init_device();
  // like the reference, construction succeeds once the model is loaded; a missing GPU surfaces
  // as the Status of the first encode call (decode / vocab keep working on the host)
  *ret_status = Status();
}

BaseEncoder::~BaseEncoder() {
  if (enc_) yttm_enc_destroy(enc_);
  if (ctx_) yttm_ctx_destroy(ctx_);
}

// fill_from_state (bpe.cpp:1667-1690)
void BaseEncoder::fill_from_state() {
  for (auto &x : bpe_state.char2id) id2char[x.second] = x.first;
  for (int i = 0; i < (int)bpe_state.rules.size(); i++)
    rule2id[((uint64_t)bpe_state.rules[i].x << 32) + bpe_state.rules[i].y] = i;
  for (auto &x : id2char) recipe[x.first] = {x.first};
  for (auto &rule : bpe_state.rules) {
    std::vector<uint32_t> r = recipe[rule.x];
    const std::vector<uint32_t> &ry = recipe[rule.y];
    r.insert(r.end(), ry.begin(), ry.end());
    recipe[rule.z] = std::move(r);
  }
  for (auto &kv : recipe) reversed_recipe[token2word(kv.second, id2char)] = kv.first;
  reversed_recipe[BOS_TOKEN] = (uint32_t)bpe_state.special_tokens.bos_id;
  reversed_recipe[EOS_TOKEN] = (uint32_t)bpe_state.special_tokens.eos_id;
}

Status BaseEncoder::init_device() {
  if (yttm_ctx_create(default_device(), &ctx_)) return Status(1, yttm_last_error(nullptr));
  std::vector<uint32_t> cp, id, xyz;
  for (auto &kv : bpe_state.char2id) { cp.push_back(kv.first); id.push_back(kv.second); }
  for (auto &r : bpe_state.rules) { xyz.push_back(r.x); xyz.push_back(r.y); xyz.push_back(r.z); }
  const SpecialTokens &st = bpe_state.special_tokens;
  if (yttm_enc_create(ctx_, cp.data(), id.data(), cp.size(), xyz.data(), bpe_state.rules.size(), st.unk_id, st.pad_id,
                      st.bos_id, st.eos_id, &enc_))
    return Status(1, ctx_err(ctx_));
  return Status();
}

int BaseEncoder::vocab_size() const {
  return (int)(bpe_state.rules.size() + bpe_state.char2id.size() + bpe_state.special_tokens.n_special_tokens());
}

Status BaseEncoder::run_device(const char *name, bool bos, bool eos, double dropout_prob, uint64_t n_sent,
                               const std::function<int()> &call, const Status &checked) const {
  if (bos && bpe_state.special_tokens.bos_id == -1)  // bpe.cpp:1702-1707
    return Status(1, "Can't add <BOS> token. Model was trained without it.");
  if (eos && bpe_state.special_tokens.eos_id == -1)
    return Status(1, "Can't add <EOS> token. Model was trained without it.");
  if (!checked.ok()) return checked;
  if (!device_status_.ok()) return device_status_;
  int rc = call();
  if (rc == 2) return Status(2, std::string(name) + ": output buffer too small");
  if (rc) return Status(1, ctx_err(ctx_));
  if (dropout_prob > 0) sentence_counter_ += n_sent;
  return Status();
}

Status BaseEncoder::encode_packed(const char *bytes, const uint64_t *offsets, uint64_t n_sent,
                                  std::vector<int32_t> *ids, std::vector<uint64_t> *id_offsets, bool bos, bool eos,
                                  bool reverse, double dropout_prob) const {
  uint64_t total_bytes = n_sent ? offsets[n_sent] - offsets[0] : 0;
  uint64_t cap = total_bytes + 3 * n_sent + 16;  // a sentence of L bytes yields at most L + 1 (+bos +eos) ids
  ids->resize(cap);
  id_offsets->resize(n_sent + 1);
  uint64_t n_out = 0;
  Status st = encode_packed_into(bytes, offsets, n_sent, ids->data(), cap, id_offsets->data(), &n_out, bos, eos, reverse,
                                 dropout_prob);
  if (!st.ok()) return st;
  ids->resize(n_out);
  return Status();
}

Status BaseEncoder::encode_packed_into(const char *bytes, const uint64_t *offsets, uint64_t n_sent, int32_t *ids,
                                       uint64_t ids_cap, uint64_t *id_offsets, uint64_t *total_ids, bool bos, bool eos,
                                       bool reverse, double dropout_prob) const {
  return run_device("encode_packed_into", bos, eos, dropout_prob, n_sent, [&] {
    return yttm_enc_run(enc_, bytes, offsets, n_sent, bos, eos, reverse, dropout_prob, dropout_seed_, sentence_counter_, ids,
                        ids_cap, id_offsets, total_ids);
  });
}

Status BaseEncoder::encode_packed_device(const char *d_bytes, const uint64_t *d_offsets, uint64_t n_bytes, uint64_t n_sent,
                                         const int32_t **d_ids, const uint64_t **d_id_offsets, uint64_t *total_ids, bool bos,
                                         bool eos, bool reverse, double dropout_prob) const {
  return run_device("encode_packed_device", bos, eos, dropout_prob, n_sent, [&] {
    return yttm_enc_run_device(enc_, d_bytes, d_offsets, n_bytes, n_sent, bos, eos, reverse, dropout_prob, dropout_seed_,
                               sentence_counter_, d_ids, d_id_offsets, total_ids);
  });
}

Status BaseEncoder::encode_spans_into(const char *bytes, const uint64_t *offsets, uint64_t n_sent, int32_t *ids,
                                      uint64_t ids_cap, uint64_t *id_offsets, uint64_t *spans, uint64_t *total_ids, bool bos,
                                      bool eos, bool reverse, double dropout_prob) const {
  return run_device("encode_spans_into", bos, eos, dropout_prob, n_sent, [&] {
    return yttm_enc_run_spans(enc_, bytes, offsets, n_sent, bos, eos, reverse, dropout_prob, dropout_seed_,
                              sentence_counter_, ids, ids_cap, id_offsets, spans, total_ids);
  });
}

Status BaseEncoder::encode_spans_device(const char *d_bytes, const uint64_t *d_offsets, uint64_t n_bytes, uint64_t n_sent,
                                        const int32_t **d_ids, const uint64_t **d_id_offsets, const uint64_t **d_spans,
                                        uint64_t *total_ids, bool bos, bool eos, bool reverse, double dropout_prob) const {
  return run_device("encode_spans_device", bos, eos, dropout_prob, n_sent, [&] {
    return yttm_enc_run_spans_device(enc_, d_bytes, d_offsets, n_bytes, n_sent, bos, eos, reverse, dropout_prob,
                                     dropout_seed_, sentence_counter_, d_ids, d_id_offsets, d_spans, total_ids);
  });
}

Status BaseEncoder::resolve_pad(int64_t pad_id, int32_t *out) const {
  if (pad_id == kModelPad) {
    if (bpe_state.special_tokens.pad_id == -1)
      return Status(1, "Can't pad: model was trained without <PAD> (pad_id = -1); pass a pad id.");
    *out = bpe_state.special_tokens.pad_id;
    return Status();
  }
  if (pad_id < INT32_MIN || pad_id > INT32_MAX)
    return Status(1, "pad_id must fit in int32. Current value of pad_id = " + std::to_string(pad_id));
  *out = (int32_t)pad_id;
  return Status();
}

Status BaseEncoder::encode_padded_into(const char *bytes, const uint64_t *offsets, uint64_t n_sent, uint64_t width,
                                       int32_t *ids, uint64_t *lengths, uint64_t *spans, bool bos, bool eos, bool reverse,
                                       double dropout_prob, int64_t pad_id) const {
  int32_t pad = 0;
  return run_device("encode_padded_into", bos, eos, dropout_prob, n_sent, [&] {
    return yttm_enc_run_padded(enc_, bytes, offsets, n_sent, bos, eos, reverse, dropout_prob, dropout_seed_,
                               sentence_counter_, width, pad, ids, lengths, spans);
  }, resolve_pad(pad_id, &pad));
}

Status BaseEncoder::encode_padded_device(const char *d_bytes, const uint64_t *d_offsets, uint64_t n_bytes, uint64_t n_sent,
                                         uint64_t width, bool with_spans, const int32_t **d_ids, const uint64_t **d_lengths,
                                         const uint64_t **d_spans, uint32_t *out_width, bool bos, bool eos, bool reverse,
                                         double dropout_prob, int64_t pad_id) const {
  int32_t pad = 0;
  return run_device("encode_padded_device", bos, eos, dropout_prob, n_sent, [&] {
    return yttm_enc_run_padded_device(enc_, d_bytes, d_offsets, n_bytes, n_sent, bos, eos, reverse, dropout_prob,
                                      dropout_seed_, sentence_counter_, width, pad, with_spans, d_ids, d_lengths, d_spans,
                                      out_width);
  }, resolve_pad(pad_id, &pad));
}

Status BaseEncoder::encode_subwords_into(const char *bytes, const uint64_t *offsets, uint64_t n_sent, uint8_t *pieces,
                                         uint64_t bytes_cap, uint64_t *piece_offsets, uint64_t pieces_cap,
                                         uint64_t *sent_offsets, uint64_t *n_pieces, uint64_t *n_bytes, bool bos, bool eos,
                                         bool reverse, double dropout_prob) const {
  return run_device("encode_subwords_into", bos, eos, dropout_prob, n_sent, [&] {
    return yttm_enc_run_subwords(enc_, bytes, offsets, n_sent, bos, eos, reverse, dropout_prob, dropout_seed_,
                                 sentence_counter_, pieces, bytes_cap, piece_offsets, pieces_cap, sent_offsets, n_pieces,
                                 n_bytes);
  });
}

Status BaseEncoder::encode_subwords_device(const char *d_bytes, const uint64_t *d_offsets, uint64_t n_bytes, uint64_t n_sent,
                                           const uint8_t **d_pieces, const uint64_t **d_piece_offsets,
                                           const uint64_t **d_sent_offsets, uint64_t *n_pieces, uint64_t *n_piece_bytes,
                                           bool bos, bool eos, bool reverse, double dropout_prob) const {
  return run_device("encode_subwords_device", bos, eos, dropout_prob, n_sent, [&] {
    return yttm_enc_run_subwords_device(enc_, d_bytes, d_offsets, n_bytes, n_sent, bos, eos, reverse, dropout_prob,
                                        dropout_seed_, sentence_counter_, d_pieces, d_piece_offsets, d_sent_offsets,
                                        n_pieces, n_piece_bytes);
  });
}

Status BaseEncoder::decode_packed_into(const int32_t *ids, const uint64_t *offsets, uint64_t n_sent, const int32_t *ignore_ids,
                                       uint64_t n_ignore, uint8_t *text, uint64_t text_cap, uint64_t *text_offsets,
                                       uint64_t *total_bytes) const {
  return run_device("decode_packed_into", false, false, 0, n_sent, [&] {
    return yttm_dec_run(enc_, ids, offsets, n_sent, ignore_ids, n_ignore, text, text_cap, text_offsets, total_bytes);
  });
}

Status BaseEncoder::decode_packed_device(const int32_t *d_ids, uint64_t n_ids, const uint64_t *d_offsets, uint64_t n_sent,
                                         const int32_t *ignore_ids, uint64_t n_ignore, const uint8_t **d_text,
                                         const uint64_t **d_text_offsets, uint64_t *total_bytes) const {
  return run_device("decode_packed_device", false, false, 0, n_sent, [&] {
    return yttm_dec_run_device(enc_, d_ids, n_ids, d_offsets, n_sent, ignore_ids, n_ignore, d_text, d_text_offsets,
                               total_bytes);
  });
}

Status BaseEncoder::encode_as_ids(const std::vector<std::string> &sentences, std::vector<std::vector<int>> *ids,
                                  bool bos, bool eos, bool reverse, double dropout_prob) const {
  std::vector<uint64_t> offs(sentences.size() + 1, 0);
  for (size_t i = 0; i < sentences.size(); i++) offs[i + 1] = offs[i] + sentences[i].size();
  std::string flat;
  flat.reserve(offs.back());
  for (auto &s : sentences) flat += s;
  std::vector<int32_t> out;
  std::vector<uint64_t> oo;
  Status st = encode_packed(flat.data(), offs.data(), sentences.size(), &out, &oo, bos, eos, reverse, dropout_prob);
  if (!st.ok()) return st;
  ids->assign(sentences.size(), std::vector<int>());
  for (size_t i = 0; i < sentences.size(); i++) (*ids)[i].assign(out.begin() + oo[i], out.begin() + oo[i + 1]);
  return Status();
}

// encode_as_subwords (bpe.cpp:1757): ids from the GPU; pieces are ids -> recipe -> UTF-8.  An
// <UNK> id carries the raw characters of its unknown run (bpe.cpp:1516-1527, 1603-1604): the
// k-th UNK of a sentence is the k-th maximal run of out-of-alphabet characters inside a word.
Status BaseEncoder::encode_as_subwords(const std::vector<std::string> &sentences,
                                       std::vector<std::vector<std::string>> *subwords, bool bos, bool eos,
                                       bool reverse, double dropout_prob) const {
  std::vector<std::vector<int>> ids;
  Status st = encode_as_ids(sentences, &ids, bos, eos, false, dropout_prob);
  if (!st.ok()) return st;
  const int unk = bpe_state.special_tokens.unk_id;
  subwords->assign(sentences.size(), std::vector<std::string>());
  for (size_t s = 0; s < sentences.size(); s++) {
    std::vector<std::string> unk_runs;
    bool has_unk = std::find(ids[s].begin(), ids[s].end(), unk) != ids[s].end();
    if (has_unk) {
      auto text = decode_utf8(sentences[s]);
      for (size_t i = 0; i < text.size();) {
        if (!is_space(text[i]) && !bpe_state.char2id.count(text[i])) {
          size_t j = i;
          while (j < text.size() && !is_space(text[j]) && !bpe_state.char2id.count(text[j])) j++;
          unk_runs.push_back(encode_utf8({text.begin() + i, text.begin() + j}));
          i = j;
        } else i++;
      }
    }
    size_t next_unk = 0;
    auto &out = (*subwords)[s];
    size_t first = 0, last = ids[s].size();
    if (bos) { out.push_back(BOS_TOKEN); first = 1; }
    if (eos) last--;
    for (size_t k = first; k < last; k++) {
      int id = ids[s][k];
      if (id == unk) out.push_back(next_unk < unk_runs.size() ? unk_runs[next_unk++] : UNK_TOKEN);
      else out.push_back(token2word(recipe.at((uint32_t)id), id2char));
    }
    if (eos) out.push_back(EOS_TOKEN);
    if (reverse) std::reverse(out.begin(), out.end());
  }
  return Status();
}

Status BaseEncoder::id_to_subword(int id, std::string *subword, bool replace_space) const {  // bpe.cpp:1774-1807
  if (id < 0 || vocab_size() <= id)
    return Status(1, "id must be in the range [0, vocab_size - 1]. Current value: vocab_size = " +
                         std::to_string(vocab_size()) + "; id=" + std::to_string(id) + ";");
  const SpecialTokens &st = bpe_state.special_tokens;
  if (st.unk_id == id) { *subword = UNK_TOKEN; return Status(); }
  if (st.pad_id == id) { *subword = PAD_TOKEN; return Status(); }
  if (st.bos_id == id) { *subword = BOS_TOKEN; return Status(); }
  if (st.eos_id == id) { *subword = EOS_TOKEN; return Status(); }
  const std::vector<uint32_t> &symbols = recipe.at((uint32_t)id);
  if (replace_space && id2char.at(symbols[0]) == SPACE_TOKEN) {
    *subword = " " + token2word({symbols.begin() + 1, symbols.end()}, id2char);
    return Status();
  }
  *subword = token2word(symbols, id2char);
  return Status();
}

int BaseEncoder::subword_to_id(const std::string &token) const {  // bpe.cpp:1809-1826
  const SpecialTokens &st = bpe_state.special_tokens;
  if (UNK_TOKEN == token) return st.unk_id;
  if (PAD_TOKEN == token) return st.pad_id;
  if (BOS_TOKEN == token) return st.bos_id;
  if (EOS_TOKEN == token) return st.eos_id;
  auto it = reversed_recipe.find(token);
  if (it != reversed_recipe.end()) return (int)it->second;
  return st.unk_id;
}

Status BaseEncoder::decode(const std::vector<int> &ids, std::string *sentence,
                           const std::unordered_set<int> *ignore_ids) const {  // bpe.cpp:1843-1861
  bool first_iter = true;
  for (int id : ids) {
    if (ignore_ids && ignore_ids->count(id)) continue;
    std::string subword;
    Status st = id_to_subword(id, &subword, true);
    if (!st.ok()) return st;
    *sentence += subword;
    if (first_iter && !sentence->empty() && sentence->at(0) == ' ') *sentence = sentence->substr(1);
    first_iter = false;
  }
  return Status();
}
Status BaseEncoder::decode(const std::vector<std::vector<int>> &ids, std::vector<std::string> *sentences,
                           const std::unordered_set<int> *ignore_ids) const {
  for (auto &s : ids) {
    std::string out;
    Status st = decode(s, &out, ignore_ids);
    if (!st.ok()) return st;
    sentences->push_back(std::move(out));
  }
  return Status();
}
Status BaseEncoder::decode(const std::vector<std::string> &data, std::vector<std::string> *sentences,
                           const std::unordered_set<int> *ignore_ids) const {
  for (auto &s : data) {
    std::stringstream stream(s);
    std::vector<int> ids;
    int x;
    while (stream >> x) ids.push_back(x);
    std::string out;
    Status st = decode(ids, &out, ignore_ids);
    if (!st.ok()) return st;
    sentences->push_back(out);
  }
  return Status();
}

std::vector<std::string> BaseEncoder::vocabulary() const {
  int n = vocab_size();
  std::vector<std::string> vocab(n);
  for (int i = 0; i < n; i++) id_to_subword(i, &vocab[i]);
  return vocab;
}

// ---------------------------------------------------------------------------------------------
// CLI loops (bpe.cpp:1896-2028): stdin/stdout framing identical to the reference
// ---------------------------------------------------------------------------------------------
void BaseEncoder::vocab_cli(bool verbose) const {
  uint32_t n_tokens = 0;
  for (auto &e : recipe) n_tokens = std::max(e.first, n_tokens);
  n_tokens = std::max(n_tokens, bpe_state.special_tokens.max_id()) + 1;
  flat_hash_map<uint32_t, std::pair<uint32_t, uint32_t>> rev;
  if (verbose)
    for (auto &r : bpe_state.rules) rev[r.z] = {r.x, r.y};
  for (uint32_t i = 0; i < n_tokens; i++) {
    std::string tz;
    id_to_subword((int)i, &tz);
    std::cout << i << "\t" << tz;
    if (verbose && rev.count(i)) {
      auto comb = rev[i];
      std::string tx, ty;
      id_to_subword((int)comb.first, &tx);
      id_to_subword((int)comb.second, &ty);
      int used = (int)decode_utf8(tz).size() + 1 + (int)decode_utf8(tx).size() + 1 + (int)decode_utf8(ty).size();
      std::cout << "=" << tx << "+" << ty;
      for (int t = 0; t < std::max(2, 50 - used); t++) std::cout << " ";
      std::cout << comb.first << "+" << comb.second;
    }
    std::cout << std::endl;
  }
}

static std::vector<std::string> read_lines(uint64_t batch_limit, uint64_t *processed) {  // utils.cpp:103-111
  std::vector<std::string> out;
  std::string s;
  while (*processed < batch_limit && std::getline(std::cin, s)) {
    *processed += s.size();
    out.push_back(std::move(s));
  }
  return out;
}
template <class T>
static void write_lines(const std::vector<std::vector<T>> &sentences, bool flush) {  // utils.h:92-103
  for (auto &sent : sentences) {
    for (auto &tok : sent) std::cout << tok << " ";
    std::cout << "\n";
  }
  if (flush) std::cout << std::flush;
}

Status BaseEncoder::encode_cli(const std::string &output_type_str, bool stream, bool bos, bool eos, bool reverse,
                               double dropout_prob) const {
  std::ios_base::sync_with_stdio(false);
  bool as_ids;
  if (output_type_str == "id") as_ids = true;
  else if (output_type_str == "subword") as_ids = false;
  else return Status(1, "output_type must be equal to \"id\" or \"subword\"");
  if (stream) {
    std::string sentence;
    while (std::getline(std::cin, sentence)) {
      if (as_ids) {
        std::vector<std::vector<int>> ids;
        Status st = encode_as_ids({sentence}, &ids, bos, eos, reverse, dropout_prob);
        if (!st.ok()) return st;
        write_lines(ids, true);
      } else {
        std::vector<std::vector<std::string>> sw;
        Status st = encode_as_subwords({sentence}, &sw, bos, eos, reverse, dropout_prob);
        if (!st.ok()) return st;
        write_lines(sw, true);
      }
    }
    return Status();
  }
  const uint64_t batch_limit = 10 * 1024 * 1024;
  uint64_t total = 0, processed = 0;
  while (true) {
    processed = 0;
    auto sentences = read_lines(batch_limit, &processed);
    if (sentences.empty()) break;
    if (as_ids) {
      std::vector<std::vector<int>> ids;
      Status st = encode_as_ids(sentences, &ids, bos, eos, reverse, dropout_prob);
      if (!st.ok()) return st;
      write_lines(ids, false);
    } else {
      std::vector<std::vector<std::string>> sw;
      Status st = encode_as_subwords(sentences, &sw, bos, eos, reverse, dropout_prob);
      if (!st.ok()) return st;
      write_lines(sw, false);
    }
    total += processed;
    std::cerr << "bytes processed: " << total << std::endl;
  }
  std::cout << std::flush;
  return Status();
}

Status BaseEncoder::decode_cli(const std::unordered_set<int> *ignore_ids) const {
  std::ios_base::sync_with_stdio(false);
  std::string line;
  while (std::getline(std::cin, line)) {
    std::vector<std::string> out;
    Status st = decode(std::vector<std::string>{line}, &out, ignore_ids);
    if (!st.ok()) return st;
    std::cout << out[0] << "\n";
  }
  std::cout << std::flush;
  return Status();
}

}  // namespace vkcom
