// bpe_host.cpp — host C++ above the C ABI: train_bpe / BaseEncoder with the reference's surface
// (youtokentome/cpp/bpe.h) and model file format (utils.cpp:50-91).  Everything data-parallel
// goes through include/yttm_b200.h to the GPU; what stays here is O(alphabet + vocab) glue:
// config validation, the coverage cut (the only floating point of training), id renaming,
// model I/O, id <-> subword tables, decode.
#include <algorithm>
#include <atomic>
#include <cassert>
#include <cerrno>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <functional>
#include <sstream>
#include <string_view>
#include <thread>

#include <fcntl.h>
#include <sys/stat.h>
#include <unistd.h>

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
// word-count tables
// ---------------------------------------------------------------------------------------------
static bool read_block(int fd, std::vector<char> &buf, size_t *got) {
  *got = 0;
  while (*got < buf.size()) {
    const ssize_t r = ::read(fd, buf.data() + *got, buf.size() - *got);
    if (r < 0 && errno == EINTR) continue;
    if (r < 0) return false;
    if (r == 0) break;
    *got += (size_t)r;
  }
  return true;
}

static Status write_tsv(const WordCounts &t, const std::string &path) {
  FILE *f = path == "-" ? stdout : std::fopen(path.c_str(), "wb");
  if (!f) return Status(1, "count_words: cannot open '" + path + "' for writing");
  std::fprintf(f, "\t%llu\n", (unsigned long long)t.separators);
  for (size_t i = 0; i + 1 < t.offsets.size(); i++) {
    std::fwrite(t.bytes.data() + t.offsets[i], 1, t.offsets[i + 1] - t.offsets[i], f);
    std::fprintf(f, "\t%llu\n", (unsigned long long)t.counts[i]);
  }
  const bool ok = std::fflush(f) == 0 && !std::ferror(f);
  if (f != stdout) std::fclose(f);
  return ok ? Status() : Status(1, "count_words: failed to write '" + path + "'");
}

Status count_words(int in_fd, const char *text, uint64_t n, const std::string &tsv_path, WordCounts *out) {
  yttm_ctx *ctx = nullptr;
  if (yttm_ctx_create(default_device(), &ctx)) return Status(1, yttm_last_error(nullptr));
  struct Destroy { yttm_ctx *c; ~Destroy() { yttm_ctx_destroy(c); } } destroy{ctx};
  if (yttm_train_feed_begin(ctx)) return Status(1, ctx_err(ctx));
  if (in_fd >= 0) {
    std::vector<char> block(FEED_BLOCK);
    for (size_t got = 0;;) {
      if (!read_block(in_fd, block, &got)) return Status(1, std::string("count_words: read failed: ") + std::strerror(errno));
      if (!got) break;
      if (yttm_train_feed(ctx, block.data(), got)) return Status(1, ctx_err(ctx));
    }
  } else {
    for (uint64_t at = 0; at < n; at += FEED_BLOCK)
      if (yttm_train_feed(ctx, text + at, std::min(FEED_BLOCK, n - at))) return Status(1, ctx_err(ctx));
  }
  uint64_t data_len = 0, n_distinct = 0, U = 0, nb = 0, seps = 0;
  if (yttm_train_feed_end(ctx, &data_len, &n_distinct)) return Status(1, ctx_err(ctx));
  if (yttm_train_fed_words(ctx, nullptr, 0, nullptr, nullptr, 0, &U, &nb, nullptr) == 1) return Status(1, ctx_err(ctx));
  std::string bytes(nb, '\0');
  std::vector<uint64_t> offs(U + 1), cnts(U);
  if (yttm_train_fed_words(ctx, reinterpret_cast<uint8_t *>(&bytes[0]), nb, offs.data(), cnts.data(), U, &U, &nb, &seps))
    return Status(1, ctx_err(ctx));
  std::vector<uint64_t> order(U);
  for (uint64_t i = 0; i < U; i++) order[i] = i;
  auto word = [&](uint64_t i) { return std::string_view(bytes.data() + offs[i], offs[i + 1] - offs[i]); };
  std::sort(order.begin(), order.end(), [&](uint64_t a, uint64_t b) {
    return cnts[a] != cnts[b] ? cnts[a] > cnts[b] : word(a) < word(b);
  });
  WordCounts &t = *out;
  t = WordCounts();
  t.bytes.reserve(nb);
  t.counts.reserve(U);
  t.offsets.reserve(U + 1);
  for (uint64_t i : order) {
    t.bytes += word(i);
    t.offsets.push_back(t.bytes.size());
    t.counts.push_back(cnts[i]);
  }
  t.separators = seps;
  t.data_len = data_len;
  return tsv_path.empty() ? Status() : write_tsv(t, tsv_path);
}

// A TSV word-count table read in blocks of FEED_BLOCK bytes and fed as word lists; the separator line ("\t<n>") may
// stand anywhere, once.
static std::string feed_tsv(yttm_ctx *ctx, const std::string &path) {
  const int fd = ::open(path.c_str(), O_RDONLY);
  if (fd < 0) return "train_from_counts: cannot open '" + path + "': " + std::strerror(errno);
  struct Closer { int fd; ~Closer() { ::close(fd); } } closer{fd};
  std::vector<char> block(FEED_BLOCK);
  std::string carry;                       // a line cut by the end of a block
  std::string wbytes;                      // the entries gathered for the next feed
  std::vector<uint64_t> woff{0}, wcnt;
  uint64_t line = 0, total = 0, seps = 0;
  bool have_seps = false;
  auto flush = [&]() -> std::string {
    if (wcnt.empty()) return "";
    if (yttm_train_feed_words(ctx, reinterpret_cast<const uint8_t *>(wbytes.data()), woff.data(), wcnt.data(),
                              wcnt.size(), 0, 0))
      return ctx_err(ctx);
    wbytes.clear(); woff.assign(1, 0); wcnt.clear();
    return "";
  };
  auto parse = [&](const char *p, size_t len) -> std::string {
    line++;
    const char *tab = static_cast<const char *>(std::memchr(p, '\t', len));
    const std::string at = path + ", line " + std::to_string(line) + ": ";
    if (!tab) return at + "no tab between the word and its count";
    const char *c = tab + 1, *e = p + len;
    if (c == e) return at + "the count is missing";
    uint64_t v = 0;
    for (const char *q = c; q < e; q++) {
      if (*q < '0' || *q > '9') return at + "the count '" + std::string(c, e) + "' is not a non-negative integer";
      const uint64_t d = (uint64_t)(*q - '0');
      if (v > (UINT64_MAX - d) / 10) return at + "the count " + std::string(c, e) + " does not fit in 64 bits";
      v = v * 10 + d;
    }
    const uint64_t wl = (uint64_t)(tab - p);
    if (!wl) {
      if (have_seps) return at + "a second separator line (empty word)";
      have_seps = true;
      seps = v;
      return "";
    }
    for (uint64_t i = 0; i < wl; i++) {
      const uint8_t b = (uint8_t)p[i];
      if (yt::is_space_byte(b) || (b == 0xe2 && i + 2 < wl && (uint8_t)p[i + 1] == 0x96 && (uint8_t)p[i + 2] == 0x81))
        return at + "the word contains a separator (a whitespace byte or U+2581)";
    }
    if (total + v < total) return at + "the counts sum past 2^64";
    total += v;
    wbytes.append(p, wl);
    woff.push_back(wbytes.size());
    wcnt.push_back(v);
    return wbytes.size() >= FEED_BLOCK ? flush() : "";
  };
  for (size_t got = 0;;) {
    if (!read_block(fd, block, &got)) return "train_from_counts: cannot read '" + path + "': " + std::strerror(errno);
    if (!got) break;
    const char *p = block.data(), *e = p + got;
    while (p < e) {
      const char *nl = static_cast<const char *>(std::memchr(p, '\n', e - p));
      if (!nl) { carry.append(p, e); break; }
      std::string err;
      if (!carry.empty()) {
        carry.append(p, nl);
        err = parse(carry.data(), carry.size());
        carry.clear();
      } else {
        err = parse(p, nl - p);
      }
      if (!err.empty()) return err;
      p = nl + 1;
    }
  }
  if (!carry.empty()) {   // a last line without its newline
    std::string err = parse(carry.data(), carry.size());
    if (!err.empty()) return err;
  }
  std::string err = flush();
  if (!err.empty()) return err;
  if (yttm_train_feed_words(ctx, nullptr, woff.data(), nullptr, 0, have_seps ? seps : total, 0)) return ctx_err(ctx);
  return "";
}

Status train_counts(const CountsInput &in, const std::string &model_path, int vocab_size, BpeConfig cfg) {
  Status status = check_config(cfg, vocab_size);
  if (!status.ok()) return status;
  print_config(in.tsv_path.empty() ? "<word counts>" : in.tsv_path, model_path, vocab_size, cfg);
  g_report = TrainReport();
  BPEState state;
  return train_on_ctx([&](yttm_ctx *ctx) -> std::string {
    std::cerr << "learning bpe from word counts..." << std::endl;
    if (yttm_train_feed_begin(ctx)) return ctx_err(ctx);
    if (!in.tsv_path.empty()) {
      std::string err = feed_tsv(ctx, in.tsv_path);
      if (!err.empty()) return err;
    } else if (yttm_train_feed_words(ctx, in.bytes, in.offsets, in.counts, in.n, in.separators, in.on_device)) {
      return ctx_err(ctx);
    }
    return yttm_train_feed_end(ctx, nullptr, nullptr) ? ctx_err(ctx) : "";
  }, vocab_size, model_path, cfg, &state);
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

Status BaseEncoder::encode_windows_device(const char *d_bytes, const uint64_t *d_offsets, uint64_t n_bytes, uint64_t n_sent,
                                          uint64_t width, uint64_t stride, bool with_spans, const int32_t **d_ids,
                                          const uint64_t **d_lengths, const uint64_t **d_sentence, const uint64_t **d_start,
                                          const uint64_t **d_spans, uint64_t *n_rows, bool bos, bool eos, bool reverse,
                                          double dropout_prob, int64_t pad_id) const {
  int32_t pad = 0;
  return run_device("encode_windows_device", bos, eos, dropout_prob, n_sent, [&] {
    return yttm_enc_run_windows_device(enc_, d_bytes, d_offsets, n_bytes, n_sent, bos, eos, reverse, dropout_prob,
                                       dropout_seed_, sentence_counter_, width, stride, pad, with_spans, d_ids, d_lengths,
                                       d_sentence, d_start, d_spans, n_rows);
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


// ---------------------------------------------------------------------------------------------
// encode_file: a file or pipe through the device's encode stream (yttm_enc_stream_* of yttm_b200.h) into .npy files or
// the text of `yttm encode --output_type id` or `--output_type subword`
// ---------------------------------------------------------------------------------------------
namespace {

// An output written under a temporary name in its directory and renamed on commit; "-" is stdout (no rename).
class OutFile {
 public:
  explicit OutFile(const char *who = "encode_file") : who_(who) {}
  ~OutFile() {
    if (fd_ >= 0 && fd_ != 1) ::close(fd_);
    if (!tmp_.empty()) ::unlink(tmp_.c_str());
  }
  Status open(const std::string &path) {
    path_ = path;
    if (path == "-") { fd_ = 1; return Status(); }
    static std::atomic<uint64_t> serial{0};
    tmp_ = path + ".part-" + std::to_string((long)::getpid()) + "-" + std::to_string(serial++);
    fd_ = ::open(tmp_.c_str(), O_WRONLY | O_CREAT | O_EXCL | O_CLOEXEC, 0666);
    if (fd_ < 0) { tmp_.clear(); return error("cannot create"); }
    return Status();
  }
  Status write(const void *data, uint64_t n) {
    const char *p = static_cast<const char *>(data);
    while (n) {
      const ssize_t k = ::write(fd_, p, std::min<uint64_t>(n, 1u << 30));
      if (k < 0 && errno == EINTR) continue;
      if (k <= 0) return error("cannot write");
      p += k;
      n -= (uint64_t)k;
    }
    return Status();
  }
  Status write_at(uint64_t at, const std::string &s) {
    if (::pwrite(fd_, s.data(), s.size(), (off_t)at) != (ssize_t)s.size()) return error("cannot write");
    return Status();
  }
  Status commit() {
    if (fd_ == 1) return Status();
    const int fd = fd_;
    fd_ = -1;
    if (::close(fd) != 0) return error("cannot write");
    if (::rename(tmp_.c_str(), path_.c_str()) != 0) return error("cannot create");
    tmp_.clear();
    return Status();
  }

 private:
  Status error(const char *what) const {
    return Status(1, std::string(who_) + ": " + what + " '" + path_ + "': " + std::strerror(errno));
  }
  const char *who_;
  std::string path_, tmp_;
  int fd_ = -1;
};

// NPY format 1.0 header of a 1-D little-endian array of n values, always 128 bytes, so that the final shape can be
// written over the first one
std::string npy_header(const char *descr, uint64_t n) {
  std::string dict = std::string("{'descr': '") + descr + "', 'fortran_order': False, 'shape': (" + std::to_string(n) +
                     ",), }";
  dict.resize(117, ' ');
  dict += '\n';
  return std::string("\x93NUMPY\x01\x00", 8) + std::string(1, (char)dict.size()) + std::string(1, '\0') + dict;
}

struct FileSink {
  bool text = false, stop = false;
  OutFile *ids = nullptr, *offsets = nullptr;  // text: `ids` holds the text
  Status st;
};

int file_sink(void *user, const void *data, uint64_t n_bytes, const uint64_t *line_ends, uint64_t n_lines) {
  auto *f = static_cast<FileSink *>(user);
  if (f->stop) return 1;
  f->st = f->ids->write(data, n_bytes);
  if (f->st.ok() && !f->text) f->st = f->offsets->write(line_ends, n_lines * 8);
  return f->st.ok() ? 0 : 1;
}

}  // namespace

Status BaseEncoder::encode_file(int in_fd, const std::string &out_path, bool text, bool bos, bool eos, bool reverse,
                                double dropout_prob, uint64_t *n_lines, uint64_t *n_ids, uint64_t *n_bytes) const {
  const int format = text ? YTTM_STREAM_TEXT : vocab_size() <= 65536 ? YTTM_STREAM_IDS16 : YTTM_STREAM_IDS32;
  return encode_file_as(in_fd, out_path, format, bos, eos, reverse, dropout_prob, n_lines, n_ids, n_bytes);
}

Status BaseEncoder::encode_file_subwords(int in_fd, const std::string &out_path, bool bos, bool eos, bool reverse,
                                         double dropout_prob, uint64_t *n_lines, uint64_t *n_ids, uint64_t *n_bytes) const {
  return encode_file_as(in_fd, out_path, YTTM_STREAM_SUBWORD, bos, eos, reverse, dropout_prob, n_lines, n_ids, n_bytes);
}

Status BaseEncoder::encode_file_as(int in_fd, const std::string &out_path, int format, bool bos, bool eos, bool reverse,
                                   double dropout_prob, uint64_t *n_lines, uint64_t *n_ids, uint64_t *n_bytes) const {
  *n_lines = *n_ids = *n_bytes = 0;
  Status st = run_device("encode_file", bos, eos, 0, 0, [] { return 0; });  // the <BOS> / <EOS> and device checks
  if (!st.ok()) return st;
  const bool text = format == YTTM_STREAM_TEXT || format == YTTM_STREAM_SUBWORD;
  if (!text && out_path == "-") return Status(1, "encode_file: the .npy form needs an output prefix, not '-'");
  const bool narrow = format == YTTM_STREAM_IDS16;
  OutFile ids_file, offsets_file;
  FileSink fs;
  fs.text = text;
  fs.ids = &ids_file;
  fs.offsets = &offsets_file;
  const char *descr = narrow ? "<u2" : "<i4";
  const uint64_t zero = 0;
  if (text) {
    if (!(st = ids_file.open(out_path)).ok()) return st;
  } else if (!(st = ids_file.open(out_path + ".ids.npy")).ok() || !(st = offsets_file.open(out_path + ".offsets.npy")).ok() ||
             !(st = ids_file.write(npy_header(descr, 0).data(), 128)).ok() ||
             !(st = offsets_file.write(npy_header("<u8", 0).data(), 128)).ok() || !(st = offsets_file.write(&zero, 8)).ok()) {
    return st;
  }
  if (yttm_enc_stream_begin(enc_, bos, eos, reverse, dropout_prob, dropout_seed_, sentence_counter_, format, file_sink, &fs))
    return Status(1, ctx_err(ctx_));
  auto failed = [&]() { return fs.st.ok() ? Status(1, ctx_err(ctx_)) : fs.st; };
  std::vector<char> block((size_t)16 << 20);
  while (true) {
    const ssize_t k = ::read(in_fd, block.data(), block.size());
    if (k < 0 && errno == EINTR) continue;
    if (k < 0) {
      st = Status(1, std::string("encode_file: cannot read the input: ") + std::strerror(errno));
      fs.stop = true;  // the stream is closed by the failure of its sink, or ends with nothing left to hand over
      uint64_t a, b, c;
      yttm_enc_stream_end(enc_, &a, &b, &c);
      return st;
    }
    if (k == 0) break;
    if (yttm_enc_stream_feed(enc_, block.data(), (uint64_t)k)) return failed();
  }
  if (yttm_enc_stream_end(enc_, n_lines, n_ids, n_bytes)) return failed();
  if (!text && (!(st = ids_file.write_at(0, npy_header(descr, *n_ids))).ok() ||
                !(st = offsets_file.write_at(0, npy_header("<u8", *n_lines + 1))).ok()))
    return st;
  if (!(st = ids_file.commit()).ok() || (!text && !(st = offsets_file.commit()).ok())) return st;
  if (dropout_prob > 0) sentence_counter_ += *n_lines;
  return Status();
}


// ---------------------------------------------------------------------------------------------
// decode_file: an .npy pair or id text through the device's decode stream (yttm_dec_stream_* of yttm_b200.h) into text
// ---------------------------------------------------------------------------------------------
namespace {

Status dec_error(const std::string &what) { return Status(1, "decode_file: " + what); }

// A 1-D little-endian .npy array (format 1.0, 2.0 or 3.0) opened for reading: its type, length and data offset.
struct NpyIn {
  int fd = -1;
  std::string path, descr;
  uint64_t n = 0, data_at = 0, item = 0;
  ~NpyIn() { if (fd >= 0) ::close(fd); }

  Status open(const std::string &p, const std::vector<std::string> &types) {
    path = p;
    fd = ::open(p.c_str(), O_RDONLY | O_CLOEXEC);
    if (fd < 0) return dec_error("cannot open '" + p + "': " + std::strerror(errno));
    struct stat sb;
    if (::fstat(fd, &sb) != 0) return dec_error("cannot read '" + p + "': " + std::strerror(errno));
    char pre[12];
    if (::pread(fd, pre, 12, 0) < 10 || std::memcmp(pre, "\x93NUMPY", 6) != 0) return bad("not an .npy file");
    const int major = (uint8_t)pre[6];
    if (major < 1 || major > 3) return bad("NPY format version " + std::to_string(major) + " is not 1, 2 or 3");
    uint64_t hlen, at;
    if (major == 1) {
      hlen = (uint8_t)pre[8] | (uint64_t)(uint8_t)pre[9] << 8;
      at = 10;
    } else {
      hlen = (uint8_t)pre[8] | (uint64_t)(uint8_t)pre[9] << 8 | (uint64_t)(uint8_t)pre[10] << 16 | (uint64_t)(uint8_t)pre[11] << 24;
      at = 12;
    }
    if (at + hlen > (uint64_t)sb.st_size || hlen > (1u << 20)) return bad("truncated header");
    std::string h(hlen, '\0');
    if (::pread(fd, &h[0], hlen, (off_t)at) != (ssize_t)hlen) return bad("truncated header");
    auto field = [&](const char *key) -> std::string {  // the text after "'key':" up to the next ',' outside brackets
      const std::string k = std::string("'") + key + "'";
      size_t i = h.find(k);
      if (i == std::string::npos) return "";
      i = h.find(':', i + k.size());
      if (i == std::string::npos) return "";
      size_t j = i + 1;
      int depth = 0;
      for (; j < h.size(); j++) {
        if (h[j] == '(') depth++;
        else if (h[j] == ')') { if (depth-- == 0) break; }
        else if ((h[j] == ',' || h[j] == '}') && depth == 0) break;
      }
      std::string v = h.substr(i + 1, j - i - 1);
      v.erase(0, v.find_first_not_of(" "));
      v.erase(v.find_last_not_of(" ") + 1);
      return v;
    };
    descr = field("descr");
    if (descr.size() >= 2 && (descr[0] == '\'' || descr[0] == '"')) descr = descr.substr(1, descr.size() - 2);
    if (std::find(types.begin(), types.end(), descr) == types.end()) {
      std::string want;
      for (auto &t : types) want += (want.empty() ? "" : " or ") + t;
      return bad("dtype '" + descr + "' is not " + want +
                 (descr == "<i8" || descr == "<u8" ? " (convert the ids with .astype(np.int32))" : ""));
    }
    item = descr == "<u2" ? 2 : descr == "<i4" ? 4 : 8;
    if (field("fortran_order") != "False") return bad("the array is in Fortran order");
    const std::string shape = field("shape");
    size_t k = 0;
    if (shape.size() < 4 || shape.front() != '(' || shape.back() != ')') return bad("shape " + shape + " is not 1-D");
    const std::string in = shape.substr(1, shape.size() - 2);
    const size_t comma = in.find(',');
    if (comma == std::string::npos || in.find_first_not_of(" ", comma + 1) != std::string::npos)
      return bad("shape " + shape + " is not 1-D");
    const std::string num = in.substr(0, comma);
    if (num.empty() || num.find_first_not_of("0123456789") != std::string::npos || num.size() > 18)
      return bad("shape " + shape + " is not 1-D");
    for (; k < num.size(); k++) n = n * 10 + (uint64_t)(num[k] - '0');
    data_at = at + hlen;
    if ((uint64_t)sb.st_size < data_at || ((uint64_t)sb.st_size - data_at) / item < n)
      return bad("truncated: " + std::to_string(n) + " values need " + std::to_string(data_at + n * item) + " bytes, the file has " +
                 std::to_string((uint64_t)sb.st_size));
    return Status();
  }
  Status read(void *dst, uint64_t first, uint64_t count) const {
    char *p = static_cast<char *>(dst);
    uint64_t at = data_at + first * item, left = count * item;
    while (left) {
      const ssize_t k = ::pread(fd, p, std::min<uint64_t>(left, 1u << 30), (off_t)at);
      if (k < 0 && errno == EINTR) continue;
      if (k <= 0) return dec_error("cannot read '" + path + "': " + (k < 0 ? std::strerror(errno) : "truncated"));
      p += k;
      at += (uint64_t)k;
      left -= (uint64_t)k;
    }
    return Status();
  }
  Status bad(const std::string &what) const { return dec_error("'" + path + "': " + what); }
};

int text_sink(void *user, const void *data, uint64_t n_bytes, const uint64_t *, uint64_t) {
  auto *f = static_cast<FileSink *>(user);
  if (f->stop) return 1;
  f->st = f->ids->write(data, n_bytes);
  return f->st.ok() ? 0 : 1;
}

}  // namespace

Status BaseEncoder::decode_file(int in_fd, const std::string &in_prefix, const std::string &out_path, bool text,
                                const std::vector<int32_t> &ignore, uint64_t *n_lines, uint64_t *n_ids,
                                uint64_t *n_bytes) const {
  *n_lines = *n_ids = *n_bytes = 0;
  Status st = run_device("decode_file", false, false, 0, 0, [] { return 0; });  // the device checks
  if (!st.ok()) return st;
  NpyIn ids_in, offs_in;
  if (!text) {
    if (!(st = ids_in.open(in_prefix + ".ids.npy", {"<u2", "<i4"})).ok()) return st;
    if (!(st = offs_in.open(in_prefix + ".offsets.npy", {"<u8"})).ok()) return st;
    if (offs_in.n == 0) return offs_in.bad("no offsets (a file of n lines has n + 1)");
  }
  OutFile out("decode_file");
  FileSink fs;
  fs.text = true;
  fs.ids = &out;
  if (!(st = out.open(out_path)).ok()) return st;
  const int format = text ? YTTM_STREAM_TEXT : ids_in.item == 2 ? YTTM_STREAM_IDS16 : YTTM_STREAM_IDS32;
  if (yttm_dec_stream_begin(enc_, format, ignore.data(), ignore.size(), text_sink, &fs)) return Status(1, ctx_err(ctx_));
  auto failed = [&]() { return fs.st.ok() ? Status(1, ctx_err(ctx_)) : fs.st; };
  auto abandon = [&](const Status &why) {  // closes the stream without handing anything more to the sink
    fs.stop = true;
    uint64_t a, b, c;
    yttm_dec_stream_end(enc_, &a, &b, &c);
    return why;
  };
  if (text) {
    std::vector<char> block((size_t)16 << 20);
    while (true) {
      const ssize_t k = ::read(in_fd, block.data(), block.size());
      if (k < 0 && errno == EINTR) continue;
      if (k < 0) return abandon(dec_error(std::string("cannot read the input: ") + std::strerror(errno)));
      if (k == 0) break;
      if (yttm_dec_stream_feed(enc_, block.data(), (uint64_t)k)) return failed();
    }
  } else {
    // blocks of up to 1 M line ends and 16 MB of ids (a longer line is read whole)
    const uint64_t L = offs_in.n - 1, max_lines = 1 << 20, max_ids = ((uint64_t)16 << 20) / ids_in.item;
    std::vector<uint64_t> ends(max_lines + 1);
    std::vector<char> ids;
    if (!(st = offs_in.read(ends.data(), 0, 1)).ok()) return abandon(st);
    if (ends[0] != 0) return abandon(offs_in.bad("offsets[0] is " + std::to_string(ends[0]) + ", not 0"));
    uint64_t done = 0, prev = 0;  // lines fed, their ids
    while (done < L) {
      const uint64_t m = std::min(max_lines, L - done);
      if (!(st = offs_in.read(ends.data(), done + 1, m)).ok()) return abandon(st);
      uint64_t k = 0;
      while (k < m) {
        uint64_t j = k, last = prev;
        for (; j < m; j++) {
          if (ends[j] < last) return abandon(offs_in.bad("offsets decrease at " + std::to_string(done + j + 1)));
          if (ends[j] > ids_in.n)
            return abandon(offs_in.bad("offsets[" + std::to_string(done + j + 1) + "] = " + std::to_string(ends[j]) +
                                       " is past the " + std::to_string(ids_in.n) + " ids"));
          if (ends[j] - prev > max_ids && j > k) break;
          last = ends[j];
        }
        ids.resize((last - prev) * ids_in.item + 1);
        if (!(st = ids_in.read(ids.data(), prev, last - prev)).ok()) return abandon(st);
        if (yttm_dec_stream_feed_ids(enc_, ids.data(), last - prev, ends.data() + k, j - k)) return failed();
        prev = last;
        k = j;
      }
      done += m;
    }
    if (prev != ids_in.n)
      return abandon(offs_in.bad("offsets[-1] = " + std::to_string(prev) + " is not the number of ids (" +
                                 std::to_string(ids_in.n) + ")"));
  }
  if (yttm_dec_stream_end(enc_, n_lines, n_ids, n_bytes)) return failed();
  return out.commit();
}

}  // namespace vkcom
