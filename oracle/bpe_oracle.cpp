// oracle/bpe_oracle.cpp — TEST INFRASTRUCTURE ONLY.
//
// A CPU restatement of the algorithm of VKCOM/YouTokenToMe's BPE trainer and encoder, written
// from the behaviour of the reference (file:line cited at each function), NOT a copy of it.
// It exists to check the CUDA product path; only tests/, __graft_entry__.smoke() and
// bench.py's cpu_baseline / --impl reference legs may load it.  The product never calls it.
//
// Parity status: PINNED.  tests/test_oracle_vs_reference.py checks this file bit-exactly
// against the unmodified reference compiled with -DDETERMINISTIC_QUEUE (oracle/_ref, built by
// oracle/Makefile) on the reference's own stress generator shape (stress_test.cpp:272-311),
// the manual case (stress_test.cpp:313-337), the golden corpora of test_manual.py:7-75 and
// committed fixtures under tests/golden/.  Exception, stated where it applies: BPE-dropout
// (dropout_prob > 0) is "parity unpinned" — the reference draws from one global, unsynchronised
// std::mt19937 (bpe.cpp:1415,1440) and is not reproducible beyond one thread, so this file and
// the CUDA path share a counter-based generator (Philox4x32-10) instead.
//
// Semantics restated (SURVEY.md §7.0):
//  * units: strict UTF-8 decode, an invalid byte is one unit (utf8.cpp:37-74);
//  * data_len counts every unit, char_cnt only valid non-space code points (bpe.cpp:839-857);
//  * alphabet by coverage cut with a double compare (bpe.cpp:316-355);
//  * removed / invalid units vanish, words close up (bpe.cpp:357-380); words are maximal
//    non-space runs, token sequence [▁] + ids, deduplicated with a count (bpe.cpp:388-418);
//  * pair statistics weighted by word count; (a,a) counted floor(run/2) (bpe.cpp:140-143,436-478);
//  * next merge = maximum under MergeCandidate::operator< (bpe.cpp:110-126);
//  * apply greedily left to right (stress_test.cpp:181-188; bpe.cpp:644-690);
//  * rename around special ids (bpe.cpp:814-837); model file as utils.cpp:50-91.
#include <algorithm>
#include <cmath>
#include <chrono>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <fstream>
#include <map>
#include <set>
#include <string>
#include <unordered_map>
#include <vector>

namespace orc {

static const uint32_t INVALID_CP = 0x0fffffffu;  // utf8.h:9
static const uint32_t SPACE_CP = 9601;           // utils.h:9  (U+2581)

// utils.cpp:99-101 : ASCII isspace in the C locale, or U+2581.
static inline bool is_space(uint32_t c) { return c == 32 || (c >= 9 && c <= 13) || c == SPACE_CP; }

// utf8.cpp:37-74 : one unit starting at p[0]; at most `size` bytes may be read.
static inline uint32_t decode_one(const uint8_t *p, uint64_t size, uint32_t *len) {
  uint8_t b0 = p[0];
  *len = 1;
  if (b0 < 0x80) return b0;
  auto cont = [](uint8_t b) { return (b & 0xc0) == 0x80; };
  auto ok_cp = [](uint32_t x) { return x < 0xd800 || (x > 0xdfff && x < 0x110000); };
  if ((b0 & 0xe0) == 0xc0) {
    if (size >= 2 && cont(p[1])) {
      uint32_t cp = ((b0 & 0x1fu) << 6) | (p[1] & 0x3fu);
      if (cp >= 0x80 && ok_cp(cp)) { *len = 2; return cp; }
    }
  } else if ((b0 & 0xf0) == 0xe0) {
    if (size >= 3 && cont(p[1]) && cont(p[2])) {
      uint32_t cp = ((b0 & 0x0fu) << 12) | ((p[1] & 0x3fu) << 6) | (p[2] & 0x3fu);
      if (cp >= 0x800 && ok_cp(cp)) { *len = 3; return cp; }
    }
  } else if ((b0 & 0xf8) == 0xf0) {
    if (size >= 4 && cont(p[1]) && cont(p[2]) && cont(p[3])) {
      uint32_t cp = ((b0 & 0x07u) << 18) | ((p[1] & 0x3fu) << 12) | ((p[2] & 0x3fu) << 6) | (p[3] & 0x3fu);
      if (cp >= 0x10000 && ok_cp(cp)) { *len = 4; return cp; }
    }
  }
  return INVALID_CP;
}

struct Rule { uint32_t x, y, z; };
struct Model {
  std::vector<std::pair<uint32_t, uint32_t>> char2id;  // (code point, id), ascending code point
  std::vector<Rule> rules;
  int unk = -1, pad = -1, bos = -1, eos = -1;
  // derived (fill())
  std::unordered_map<uint32_t, uint32_t> c2i;
  std::unordered_map<uint64_t, uint32_t> rule2id;  // bpe.cpp:1672-1674
  uint32_t space_id = 0;
  void fill() {
    c2i.clear(); rule2id.clear();
    for (auto &p : char2id) c2i[p.first] = p.second;
    for (size_t i = 0; i < rules.size(); i++) rule2id[((uint64_t)rules[i].x << 32) | rules[i].y] = (uint32_t)i;
    space_id = c2i.count(SPACE_CP) ? c2i[SPACE_CP] : 0;
  }
  int n_special() const { return (unk != -1) + (pad != -1) + (bos != -1) + (eos != -1); }
  bool taken(int id) const { return id == unk || id == pad || id == bos || id == eos; }
};

// MergeCandidate::operator< (bpe.cpp:110-126): a < b  <=>  b is preferred.
struct Cand {
  uint64_t cnt; uint32_t x, y;
  bool operator<(const Cand &o) const {
    if (cnt != o.cnt) return cnt < o.cnt;
    uint32_t mn = std::min(x, y), mx = std::max(x, y), omn = std::min(o.x, o.y), omx = std::max(o.x, o.y);
    if (mx != omx) return mx > omx;
    if (mn != omn) return mn > omn;
    return x < o.x;
  }
};

static inline uint64_t key(uint32_t a, uint32_t b) { return ((uint64_t)a << 32) | b; }

// Pair multiset of one word under the run rule (bpe.cpp:465-475; stress_test.cpp:153-158).
template <class F>
static void for_each_pair(const std::vector<uint32_t> &w, F f) {
  size_t n = w.size(), i = 0;
  while (i < n) {
    size_t j = i;
    while (j < n && w[j] == w[i]) j++;
    uint64_t run = j - i;
    if (run >= 2) f(key(w[i], w[i]), run / 2);
    if (j < n) f(key(w[i], w[j]), (uint64_t)1);
    i = j;
  }
}

struct TrainStats { uint64_t data_len = 0, n_words = 0, n_unique = 0, n_tokens = 0, n_merges = 0; };

struct MergeRule { uint32_t x, y, z; uint64_t cnt; };  // cnt: count of (x, y) at merge time

// Phases 3-4 over a list of words (bpe.cpp:436-478, main :1121-1282, worker :601-811): pair counts under the run
// rule weighted by wfreq, then up to max_merges merges with new ids first_new_id, first_new_id + 1, ...  `words` is
// rewritten in place; *live receives the pair counts after the last merge (zero counts included).  Equal words may
// appear more than once: their statistics add up.  A word of fewer than 2 tokens carries no pair.
static void merge_words(std::vector<std::vector<uint32_t>> &words, const std::vector<uint64_t> &wfreq,
                        uint32_t first_new_id, uint64_t max_merges, std::vector<MergeRule> *rules,
                        std::unordered_map<uint64_t, uint64_t> *live) {
  std::unordered_map<uint64_t, uint64_t> cnt;
  std::unordered_map<uint64_t, std::vector<uint32_t>> where;  // pair -> words that (once) held it
  std::set<Cand> order;                                        // all pairs with cnt > 0
  for (uint32_t wi = 0; wi < words.size(); wi++) {
    for_each_pair(words[wi], [&](uint64_t k, uint64_t c) {
      cnt[k] += c * wfreq[wi];
      auto &v = where[k];
      if (v.empty() || v.back() != wi) v.push_back(wi);
    });
  }
  for (auto &kv : cnt) order.insert({kv.second, (uint32_t)(kv.first >> 32), (uint32_t)kv.first});

  auto add = [&](uint64_t k, int64_t d) {
    if (d == 0) return;
    uint64_t &c = cnt[k];
    if (c) order.erase({c, (uint32_t)(k >> 32), (uint32_t)k});
    c = (uint64_t)((int64_t)c + d);
    if (c) order.insert({c, (uint32_t)(k >> 32), (uint32_t)k});
  };

  std::vector<uint32_t> nw;
  std::unordered_map<uint64_t, int64_t> delta;  // count changes of one merge, applied before the next election
  for (uint64_t m = 0; m < max_merges; m++) {
    if (order.empty()) break;  // "WARNING merged only" (bpe.cpp:1137-1145)
    Cand best = *order.rbegin();
    uint32_t x = best.x, y = best.y, z = first_new_id + (uint32_t)m;
    rules->push_back({x, y, z, best.cnt});
    std::vector<uint32_t> affected;
    affected.swap(where[key(x, y)]);
    delta.clear();
    for (uint32_t wi : affected) {
      auto &w = words[wi];
      nw.clear();
      bool any = false;
      for (size_t i = 0; i < w.size();) {  // greedy left to right (stress_test.cpp:181-188)
        if (i + 1 < w.size() && w[i] == x && w[i + 1] == y) { nw.push_back(z); i += 2; any = true; }
        else nw.push_back(w[i++]);
      }
      if (!any) continue;
      int64_t f = (int64_t)wfreq[wi];
      for_each_pair(w, [&](uint64_t k, uint64_t c) { delta[k] -= (int64_t)c * f; });
      w = nw;
      for_each_pair(w, [&](uint64_t k, uint64_t c) {
        delta[k] += (int64_t)c * f;
        auto &v = where[k];
        if (v.empty() || v.back() != wi) v.push_back(wi);
      });
    }
    for (auto &kv : delta) add(kv.first, kv.second);
  }
  if (live) live->swap(cnt);
}

// learn_bpe_from_string (bpe.cpp:859-1293) without the thread choreography.
// Returns "" or an error message (bpe.cpp:1053-1062).
static std::string train(const uint8_t *text, uint64_t n, int vocab_size, double coverage, Model *m, TrainStats *st) {
  // phase 1: unit count + char histogram (bpe.cpp:839-857)
  std::map<uint32_t, uint64_t> char_cnt;
  uint64_t data_len = 0;
  for (uint64_t p = 0; p < n;) {
    uint32_t len, cp = decode_one(text + p, n - p, &len);
    data_len++;
    if (cp != INVALID_CP && !is_space(cp)) char_cnt[cp]++;
    p += len;
  }
  // alphabet (bpe.cpp:316-355): ascending (count, cp); drop rarest while the rest still covers.
  std::vector<std::pair<uint64_t, uint32_t>> freq;
  for (auto &kv : char_cnt) freq.emplace_back(kv.second, kv.first);
  std::sort(freq.begin(), freq.end());
  uint64_t cur = 0, n_removed = 0;
  for (; cur < freq.size() && (double)(data_len - n_removed - freq[cur].first) > (double)data_len * coverage; cur++)
    n_removed += freq[cur].first;
  std::unordered_map<uint32_t, uint32_t> c2i;  // internal ids
  uint32_t used = (uint32_t)m->n_special();
  c2i[SPACE_CP] = used++;
  for (int64_t i = (int64_t)freq.size() - 1; i >= (int64_t)cur; i--) c2i[freq[i].second] = used++;
  if ((int64_t)used > (int64_t)vocab_size)
    return "Incorrect arguments. Vocabulary size too small. Set vocab_size>=" + std::to_string(used) +
           ".  Current value for vocab_size=" + std::to_string(vocab_size);

  // phase 2: words (bpe.cpp:357-418).  Removed and invalid units emit nothing.
  std::map<std::vector<uint32_t>, uint64_t> wmap;
  {
    std::vector<uint32_t> w;
    uint64_t nwords = 0;
    auto flush = [&]() {
      if (w.size() > 1) { wmap[w]++; nwords++; }
      w.clear();
    };
    for (uint64_t p = 0; p < n;) {
      uint32_t len, cp = decode_one(text + p, n - p, &len);
      p += len;
      if (cp == INVALID_CP) continue;
      if (is_space(cp)) { flush(); continue; }
      auto it = c2i.find(cp);
      if (it == c2i.end()) continue;  // removed char
      if (w.empty()) w.push_back(c2i[SPACE_CP]);
      w.push_back(it->second);
    }
    flush();
    if (st) st->n_words = nwords;
  }
  std::vector<std::vector<uint32_t>> words;
  std::vector<uint64_t> wfreq;
  for (auto &kv : wmap) { words.push_back(kv.first); wfreq.push_back(kv.second); }
  wmap.clear();

  uint64_t ntok = 0;
  for (auto &w : words) ntok += w.size();
  if (st) { st->data_len = data_len; st->n_unique = words.size(); st->n_tokens = ntok; }

  // phases 3-4: pair counts + merge loop
  std::vector<MergeRule> rules;
  merge_words(words, wfreq, used, vocab_size > (int)used ? (uint64_t)(vocab_size - (int)used) : 0, &rules, nullptr);
  if (st) st->n_merges = rules.size();

  // rename_tokens (bpe.cpp:814-837)
  std::vector<uint32_t> ren(vocab_size + 8, 0);
  {
    uint32_t c = (uint32_t)m->n_special();
    for (uint32_t i = 0; i < (uint32_t)vocab_size; i++)
      if (!m->taken((int)i)) ren[c++] = i;
  }
  m->char2id.clear();
  for (auto &kv : c2i) m->char2id.emplace_back(kv.first, ren[kv.second]);
  std::sort(m->char2id.begin(), m->char2id.end());
  m->rules.clear();
  for (auto &r : rules) m->rules.push_back({ren[r.x], ren[r.y], ren[r.z]});
  m->fill();
  return "";
}

// ---------------------------------------------------------------- Philox4x32-10 (dropout only)
static inline void philox(uint32_t k0, uint32_t k1, uint32_t c[4]) {
  for (int r = 0; r < 10; r++) {
    uint64_t p0 = (uint64_t)0xD2511F53u * c[0], p1 = (uint64_t)0xCD9E8D57u * c[2];
    uint32_t n0 = (uint32_t)(p1 >> 32) ^ c[1] ^ k0, n1 = (uint32_t)p1;
    uint32_t n2 = (uint32_t)(p0 >> 32) ^ c[3] ^ k1, n3 = (uint32_t)p0;
    c[0] = n0; c[1] = n1; c[2] = n2; c[3] = n3;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
}
// One Bernoulli(skip) draw: counter = (sentence index lo/hi, byte offset of the word in the
// sentence, draw number); key = seed.  skip <=> r < ceil(p * 2^32), i.e. r / 2^32 < p.
static inline bool drop_draw(uint64_t seed, uint64_t sent, uint32_t word_off, uint32_t draw, uint64_t thresh) {
  uint32_t c[4] = {(uint32_t)sent, (uint32_t)(sent >> 32), word_off, draw};
  philox((uint32_t)seed, (uint32_t)(seed >> 32), c);
  return (uint64_t)c[0] < thresh;
}

// encode_sentence (bpe.cpp:1455-1632), ids only.  Merge order: minimum rule index, leftmost
// first (MergeEvent2::operator< bpe.cpp:1475-1478) — equal to decode_slow (stress_test.cpp:195-270).
static void encode(const Model &m, const uint8_t *s, uint64_t n, bool bos, bool eos, bool reverse, double dropout,
                   uint64_t seed, uint64_t sent_index, std::vector<int32_t> *out) {
  size_t out0 = out->size();
  if (bos) out->push_back(m.bos);
  // decode_utf8 (utf8.cpp:111-128) drops invalid bytes.  For the RNG key every kept unit remembers the byte offset
  // at which its WORD starts on the raw bytes: the first unit - valid or not - of the maximal run of non-space
  // units it belongs to (an invalid byte is a non-space unit: "\xc0\xafabc" is one word starting at offset 0).
  std::vector<uint32_t> cps; std::vector<uint32_t> offs;
  bool in_word = false;
  uint32_t word_start = 0;
  for (uint64_t p = 0; p < n;) {
    uint32_t len, cp = decode_one(s + p, n - p, &len);
    const bool space = cp != INVALID_CP && is_space(cp);
    if (space) in_word = false;
    else if (!in_word) { in_word = true; word_start = (uint32_t)p; }
    if (cp != INVALID_CP) { cps.push_back(cp); offs.push_back(space ? (uint32_t)p : word_start); }
    p += len;
  }
  while (!cps.empty() && is_space(cps.back())) { cps.pop_back(); offs.pop_back(); }  // bpe.cpp:1500
  const uint32_t UNK_BASE = 1000000000u;  // bpe.cpp:1503
  uint64_t thresh = dropout <= 0 ? 0 : (uint64_t)std::ceil(std::min(dropout, 1.0) * 4294967296.0);  // r / 2^32 < p
  std::vector<uint32_t> t;
  for (size_t i = 0; i < cps.size();) {
    while (i < cps.size() && is_space(cps[i])) i++;
    if (i >= cps.size()) break;
    uint32_t word_off = offs[i];
    t.clear();
    t.push_back(m.space_id);
    uint32_t unk_next = UNK_BASE;
    while (i < cps.size() && !is_space(cps[i])) {
      auto it = m.c2i.find(cps[i]);
      if (it == m.c2i.end()) {  // maximal unknown run -> one pseudo token (bpe.cpp:1516-1527)
        while (i < cps.size() && !is_space(cps[i]) && !m.c2i.count(cps[i])) i++;
        t.push_back(unk_next++);
      } else { t.push_back(it->second); i++; }
    }
    if (thresh == 0) {
      for (;;) {  // minimum rule index, leftmost first
        int best = -1; uint32_t best_r = 0;
        for (int p = 0; p + 1 < (int)t.size(); p++) {
          auto it = m.rule2id.find(key(t[p], t[p + 1]));
          if (it != m.rule2id.end() && (best < 0 || it->second < best_r)) { best = p; best_r = it->second; }
        }
        if (best < 0) break;
        t[best] = m.rules[best_r].z;
        t.erase(t.begin() + best + 1);
      }
    } else {
      // DropoutQueue + the caller's loop, restated directly (bpe.cpp:1417-1453, 1549-1589): a set of
      // events (rule, node) ordered like MergeEvent2; pop() draws once per event in order, returns
      // the first one not skipped (skipped ones stay queued), or "empty" if all were skipped;
      // a popped event whose pair no longer matches its rule is stale and simply dropped.
      const int nn = (int)t.size();
      std::vector<int> nxt(nn), prv(nn);
      std::vector<bool> dead(nn, false);
      for (int i = 0; i < nn; i++) { nxt[i] = i + 1 < nn ? i + 1 : -1; prv[i] = i - 1; }
      std::set<std::pair<uint32_t, int>> events;
      auto push_if_rule = [&](int p) {
        auto it = m.rule2id.find(key(t[p], t[nxt[p]]));
        if (it != m.rule2id.end()) events.insert({it->second, p});
      };
      for (int i = 0; i + 1 < nn; i++) push_if_rule(i);
      uint32_t draw = 0;
      for (;;) {
        auto acc = events.end();
        for (auto it = events.begin(); it != events.end(); ++it)
          if (!drop_draw(seed, sent_index, word_off, draw++, thresh)) { acc = it; break; }
        if (acc == events.end()) break;
        uint32_t rule = acc->first; int p1 = acc->second;
        events.erase(acc);
        int p2 = dead[p1] ? -1 : nxt[p1];
        if (dead[p1] || p2 == -1 || t[p1] != m.rules[rule].x || t[p2] != m.rules[rule].y) continue;  // stale
        int pl = prv[p1], p3 = nxt[p2];
        dead[p2] = true;
        t[p1] = m.rules[rule].z;
        nxt[p1] = p3;
        if (p3 != -1) prv[p3] = p1;
        if (pl != -1) push_if_rule(pl);
        if (p3 != -1) push_if_rule(p1);
      }
      std::vector<uint32_t> live;
      for (int i = 0; i != -1; i = nxt[i]) live.push_back(t[i]);
      t.swap(live);
    }
    // The reference starts its output at the first node whose token id is not 0 (dead nodes carry id 0,
    // bpe.cpp:1591-1596): when U+2581 itself has id 0 (no special token sits at 0, e.g. pad_id = -1) a word-initial
    // "▁" that was never merged is silently dropped.  Reproduced, not fixed.
    const size_t first = (m.space_id == 0 && !t.empty() && t[0] == 0) ? 1 : 0;
    for (size_t k = first; k < t.size(); k++) out->push_back(t[k] >= UNK_BASE ? m.unk : (int32_t)t[k]);
  }
  if (eos) out->push_back(m.eos);
  if (reverse) std::reverse(out->begin() + out0, out->end());
}

static bool save(const Model &m, const std::string &path) {  // utils.cpp:50-66, :10-13
  std::ofstream f(path);
  if (!f) return false;
  f << m.char2id.size() << " " << m.rules.size() << "\n";
  for (auto &p : m.char2id) f << p.first << " " << p.second << "\n";
  for (auto &r : m.rules) f << r.x << " " << r.y << " " << r.z << "\n";
  f << m.unk << " " << m.pad << " " << m.bos << " " << m.eos << "\n";
  return true;
}
static bool load(Model *m, const std::string &path) {  // utils.cpp:68-91
  std::ifstream f(path);
  if (!f) return false;
  int n, r;
  f >> n >> r;
  m->char2id.clear(); m->rules.clear();
  for (int i = 0; i < n; i++) { uint32_t a, b; f >> a >> b; m->char2id.emplace_back(a, b); }
  for (int i = 0; i < r; i++) { Rule q; f >> q.x >> q.y >> q.z; m->rules.push_back(q); }
  f >> m->unk >> m->pad >> m->bos >> m->eos;
  std::sort(m->char2id.begin(), m->char2id.end());
  m->fill();
  return true;
}

}  // namespace orc

namespace {
double now_s() { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); }
void set_err(char *err, int errlen, const std::string &s) {
  if (err && errlen > 0) { std::strncpy(err, s.c_str(), errlen - 1); err[errlen - 1] = 0; }
}
struct Handle { orc::Model m; std::vector<int32_t> ids; std::vector<uint64_t> offs; };
// what the last orc_train_words left behind (orc_words_state)
struct WordsState {
  std::vector<std::vector<uint32_t>> words;
  std::vector<uint64_t> wfreq;
  std::unordered_map<uint64_t, uint64_t> live;
};
WordsState g_words;
}  // namespace

extern "C" {

int orc_train_memory(const char *text, uint64_t n, const char *model_path, int vocab_size, double coverage,
                     int pad_id, int unk_id, int bos_id, int eos_id, double *seconds, uint64_t *stats5, char *err,
                     int errlen) {
  orc::Model m; m.pad = pad_id; m.unk = unk_id; m.bos = bos_id; m.eos = eos_id;
  orc::TrainStats st;
  double t0 = now_s();
  std::string e = orc::train((const uint8_t *)text, n, vocab_size, coverage, &m, &st);
  if (seconds) *seconds = now_s() - t0;
  if (stats5) { stats5[0] = st.data_len; stats5[1] = st.n_words; stats5[2] = st.n_unique; stats5[3] = st.n_tokens; stats5[4] = st.n_merges; }
  if (!e.empty()) { set_err(err, errlen, e); return 1; }
  if (model_path && *model_path && !orc::save(m, model_path)) { set_err(err, errlen, "cannot write model"); return 1; }
  return 0;
}

// The merge loop of training on given words (the words-in form of phases 3-4): word i = tokens[offsets[i],
// offsets[i+1]) with frequency freq[i].  Up to max_merges rules (x, y, z) into out_rules (3 per merge) and the
// count of (x, y) at merge time into out_freqs; *n_done = merges made.  The words and the pair table after the
// merges stay for orc_words_state.
int orc_train_words(const uint32_t *tokens, uint64_t n_tokens, const uint32_t *offsets, const uint64_t *freq,
                    uint64_t n_words, uint32_t first_new_id, uint32_t max_merges, uint32_t *out_rules,
                    uint64_t *out_freqs, uint32_t *n_done) {
  g_words = WordsState();
  g_words.words.resize(n_words);
  g_words.wfreq.assign(freq, freq + n_words);
  for (uint64_t i = 0; i < n_words; i++) {
    if (offsets[i] > offsets[i + 1] || offsets[i + 1] > n_tokens) return 1;
    g_words.words[i].assign(tokens + offsets[i], tokens + offsets[i + 1]);
  }
  std::vector<orc::MergeRule> rules;
  orc::merge_words(g_words.words, g_words.wfreq, first_new_id, max_merges, &rules, &g_words.live);
  for (size_t i = 0; i < rules.size(); i++) {
    out_rules[3 * i] = rules[i].x; out_rules[3 * i + 1] = rules[i].y; out_rules[3 * i + 2] = rules[i].z;
    out_freqs[i] = rules[i].cnt;
  }
  *n_done = (uint32_t)rules.size();
  return 0;
}

// State after the last orc_train_words: its words (same order, with their frequencies) and the live pair table
// (key = x << 32 | y, count > 0).  With tokens == nullptr only the sizes are returned.
int orc_words_state(uint32_t *tokens, uint64_t *offsets, uint64_t *freq, uint64_t *keys, uint64_t *counts,
                    uint64_t *n_words, uint64_t *n_tokens, uint64_t *n_pairs) {
  uint64_t nt = 0, np = 0;
  for (auto &w : g_words.words) nt += w.size();
  for (auto &kv : g_words.live) np += kv.second != 0;
  *n_words = g_words.words.size(); *n_tokens = nt; *n_pairs = np;
  if (!tokens) return 0;
  uint64_t p = 0;
  for (size_t i = 0; i < g_words.words.size(); i++) {
    offsets[i] = p;
    for (uint32_t t : g_words.words[i]) tokens[p++] = t;
    freq[i] = g_words.wfreq[i];
  }
  offsets[g_words.words.size()] = p;
  uint64_t q = 0;
  for (auto &kv : g_words.live)
    if (kv.second) { keys[q] = kv.first; counts[q] = kv.second; q++; }
  return 0;
}

void *orc_encoder_new(const char *model_path, char *err, int errlen) {
  auto *h = new Handle();
  if (!orc::load(&h->m, model_path)) { set_err(err, errlen, std::string("Can not open file with model: ") + model_path); delete h; return nullptr; }
  return h;
}
void orc_encoder_free(void *h) { delete static_cast<Handle *>(h); }
int orc_vocab_size(void *hv) { auto *h = static_cast<Handle *>(hv); return (int)(h->m.rules.size() + h->m.char2id.size() + h->m.n_special()); }

int orc_encode_ids(void *hv, const char *bytes, const uint64_t *offsets, uint64_t n_sent, int bos, int eos, int reverse,
                   double dropout, uint64_t seed, uint64_t first_sentence_index, double *seconds, uint64_t *total_ids,
                   char *err, int errlen) {
  auto *h = static_cast<Handle *>(hv);
  if (bos && h->m.bos == -1) { set_err(err, errlen, "Can't add <BOS> token. Model was trained without it."); return 1; }
  if (eos && h->m.eos == -1) { set_err(err, errlen, "Can't add <EOS> token. Model was trained without it."); return 1; }
  h->ids.clear(); h->offs.assign(1, 0);
  double t0 = now_s();
  for (uint64_t i = 0; i < n_sent; i++) {
    orc::encode(h->m, (const uint8_t *)bytes + offsets[i], offsets[i + 1] - offsets[i], bos, eos, reverse, dropout, seed,
                first_sentence_index + i, &h->ids);
    h->offs.push_back(h->ids.size());
  }
  if (seconds) *seconds = now_s() - t0;
  if (total_ids) *total_ids = h->ids.size();
  return 0;
}
void orc_result_ids(void *hv, int32_t *out_ids, uint64_t *out_offsets) {
  auto *h = static_cast<Handle *>(hv);
  std::memcpy(out_ids, h->ids.data(), h->ids.size() * 4);
  std::memcpy(out_offsets, h->offs.data(), h->offs.size() * 8);
}

}  // extern "C"
