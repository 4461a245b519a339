// tests/emul/emul.cpp — TEST HARNESS ONLY (never shipped, never a fallback).
//
// Runs the kernels' building blocks of youtokentome_b200/csrc/bpe_core.cuh — the SAME source the
// sm_90a kernels compile — sequentially on the CPU, following the kernels' control flow
// (per-byte unit/word detection, byte-keyed word dedup, run-rule pair counting, arg-max by
// pair_prio, has_pair / rewrite_word / whole-word recount, encode_word).  tests/test_emul_cpu.py
// compares the result with the oracle, so logic errors in the device functions are caught in
// the build container, which has no GPU.
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <fstream>
#include <map>
#include <string>
#include <unordered_map>
#include <vector>

#include "../../youtokentome_b200/csrc/bpe_core.cuh"

using namespace yt;

namespace {
struct Rule { uint32_t x, y, z; };
}

extern "C" {

// returns 0 ok, 1 vocab too small
int emul_train(const char *text_c, uint64_t n, int vocab_size, double coverage, int pad, int unk, int bos, int eos,
               const char *model_path, uint64_t *stats4) {
  const uint8_t *s = (const uint8_t *)text_c;
  // ---- char_hist_kernel
  std::map<uint32_t, uint64_t> hist;
  uint64_t data_len = 0;
  for (uint64_t p = 0; p < n; p++) {
    if (!is_unit_start(s, p, 0, n)) continue;
    data_len++;
    uint32_t len, cp = decode_unit(s, p, n, &len);
    if (cp == INVALID_CP || is_space_cp(cp)) continue;
    hist[cp]++;
  }
  // ---- host alphabet (bpe_host.cpp compute_alphabet_helper)
  int n_special = (pad != -1) + (unk != -1) + (bos != -1) + (eos != -1);
  std::vector<std::pair<uint64_t, uint32_t>> freq;
  for (auto &kv : hist) freq.emplace_back(kv.second, kv.first);
  std::sort(freq.begin(), freq.end());
  uint64_t cur = 0, removed = 0;
  for (; cur < freq.size() && (double)(data_len - removed - freq[cur].first) > (double)data_len * coverage; cur++)
    removed += freq[cur].first;
  std::vector<uint32_t> cp2id(CP_LIMIT, NO_ID);
  std::map<uint32_t, uint32_t> char2id;
  uint32_t used = n_special;
  uint32_t space_id = used++;
  char2id[SPACE_CP] = space_id;
  for (int64_t i = (int64_t)freq.size() - 1; i >= (int64_t)cur; i--) { cp2id[freq[i].second] = used; char2id[freq[i].second] = used++; }
  if ((int64_t)used > vocab_size) return 1;
  // ---- word_insert_kernel (byte-keyed dedup; representative = first position)
  std::map<std::string, std::pair<uint64_t, uint64_t>> words;  // bytes -> (pos, count)
  uint64_t occ = 0;
  for (uint64_t p = 0; p < n; p++) {
    if (!word_start_at(s, p, 0, n)) continue;
    occ++;
    uint64_t q = p;
    uint32_t l;
    while (q < n && !space_at(s, q, n, &l)) q++;
    std::string key((const char *)s + p, q - p);
    auto it = words.find(key);
    if (it == words.end()) words[key] = {p, 1};
    else it->second.second++;
  }
  // ---- word_tokens_kernel
  std::vector<uint32_t> tok;
  std::vector<uint32_t> off(1, 0);
  std::vector<uint64_t> wfreq;
  for (auto &kv : words) {
    uint64_t q = kv.second.first;
    uint32_t l;
    std::vector<uint32_t> w(1, space_id);
    while (q < n && !space_at(s, q, n, &l)) {
      uint32_t cp = decode_unit(s, q, n, &l);
      q += l;
      if (cp == INVALID_CP || cp2id[cp] == NO_ID) continue;
      w.push_back(cp2id[cp]);
    }
    if (w.size() < 2) continue;
    tok.insert(tok.end(), w.begin(), w.end());
    off.push_back((uint32_t)tok.size());
    wfreq.push_back(kv.second.second);
  }
  uint64_t n_words = wfreq.size();
  if (stats4) { stats4[0] = data_len; stats4[1] = occ; stats4[2] = n_words; stats4[3] = tok.size(); }
  // ---- pair_hist_kernel
  std::unordered_map<uint64_t, int64_t> cnt;
  for (uint64_t w = 0; w < n_words; w++)
    for_each_pair(tok.data() + off[w], off[w + 1] - off[w], [&](uint64_t k, uint64_t m) { cnt[k] += (int64_t)(m * wfreq[w]); });
  // ---- merge_loop_kernel
  std::vector<Rule> rules;
  while ((int64_t)used < vocab_size) {
    uint64_t bc = 0, bp = 0, bk = 0;
    for (auto &kv : cnt) {
      if (kv.second <= 0) continue;
      uint64_t c = (uint64_t)kv.second, pr = pair_prio((uint32_t)(kv.first >> 32), (uint32_t)kv.first);
      if (c > bc || (c == bc && pr > bp)) { bc = c; bp = pr; bk = kv.first; }
    }
    if (bc == 0) break;
    uint32_t x = (uint32_t)(bk >> 32), y = (uint32_t)bk, z = used++;
    rules.push_back({x, y, z});
    cnt[bk] = 0;
    for (uint64_t w = 0; w < n_words; w++) {
      uint32_t *t = tok.data() + off[w];
      uint32_t cap = off[w + 1] - off[w];
      if (!has_pair(t, cap, x, y)) continue;
      int64_t f = (int64_t)wfreq[w];
      for_each_pair(t, cap, [&](uint64_t k, uint64_t m) { if (k != bk) cnt[k] -= (int64_t)m * f; });
      rewrite_word(t, cap, x, y, z);
      for_each_pair(t, cap, [&](uint64_t k, uint64_t m) { cnt[k] += (int64_t)m * f; });
    }
  }
  for (auto &kv : cnt) if (kv.second < 0) return 3;  // a count went negative: logic error
  // ---- rename + dump (bpe_host.cpp)
  std::vector<uint32_t> ren(vocab_size + 8, 0);
  {
    uint32_t c = n_special;
    for (int i = 0; i < vocab_size; i++)
      if (!(i == pad || i == unk || i == bos || i == eos)) ren[c++] = i;
  }
  std::ofstream f(model_path);
  f << char2id.size() << " " << rules.size() << "\n";
  for (auto &kv : char2id) f << kv.first << " " << ren[kv.second] << "\n";
  for (auto &r : rules) f << ren[r.x] << " " << ren[r.y] << " " << ren[r.z] << "\n";
  f << unk << " " << pad << " " << bos << " " << eos << "\n";
  return 0;
}

// encode with the kernels' logic; out_ids must hold n_bytes + 3 * n_sent entries
int emul_encode(const char *model_path, const char *bytes_c, const uint64_t *offs, uint64_t n_sent, int bos, int eos,
                int reverse, double dropout, uint64_t seed, uint64_t first_index, int32_t *out_ids, uint64_t *out_offs) {
  std::ifstream f(model_path);
  if (!f) return 1;
  int nc, nr;
  f >> nc >> nr;
  std::vector<uint32_t> cp2id(CP_LIMIT, NO_ID);
  uint32_t space_id = 0;
  for (int i = 0; i < nc; i++) { uint32_t a, b; f >> a >> b; cp2id[a] = b; if (a == SPACE_CP) space_id = b; }
  std::unordered_map<uint64_t, std::pair<uint32_t, uint32_t>> rt;
  std::vector<uint32_t> zs(nr + 1, 0);
  for (int i = 0; i < nr; i++) { uint32_t x, y, z; f >> x >> y >> z; rt[pair_key(x, y)] = {(uint32_t)i, z}; zs[i] = z; }
  int unk_id, pad_id, bos_id, eos_id;
  f >> unk_id >> pad_id >> bos_id >> eos_id;
  auto rank = [&](uint32_t a, uint32_t b, uint32_t *z) -> uint32_t {
    if ((a | b) & UNK_FLAG) return NO_RANK_V;
    auto it = rt.find(pair_key(a, b));
    if (it == rt.end()) return NO_RANK_V;
    *z = it->second.second;
    return it->second.first;
  };
  const uint8_t *s = (const uint8_t *)bytes_c;
  uint64_t thresh = dropout <= 0 ? 0 : (uint64_t)std::ceil(std::min(dropout, 1.0) * 4294967296.0);  // as enc_device
  uint64_t pos = 0;
  for (uint64_t si = 0; si < n_sent; si++) {
    out_offs[si] = pos;
    uint64_t lo = offs[si] - offs[0], hi = offs[si + 1] - offs[0], len = hi - lo;
    std::vector<int32_t> slots(len + 3, -1);
    std::vector<uint32_t> ranks(len + 3, 0), zcache(len + 3, 0), auxv(6 * (len + 3), 0);
    if (bos) slots[0] = bos_id;
    if (eos) slots[len + 2] = eos_id;
    for (uint64_t p = lo; p < hi; p++) {
      if (!word_start_at(s, p, lo, hi)) continue;
      int32_t *t = slots.data() + 1 + (p - lo);
      uint32_t *r = ranks.data() + 1 + (p - lo);
      uint32_t *aux = auxv.data() + 6 * (1 + (p - lo));
      uint32_t owned;
      uint32_t n = encode_word(s, p, lo, hi, cp2id.data(), space_id, rank, thresh ? nullptr : zcache.data() + 1 + (p - lo), thresh, seed, first_index + si, t, r, aux, &owned);
      for (uint32_t i = 0; i < n; i++) if ((uint32_t)t[i] & UNK_FLAG) t[i] = unk_id;
      for (uint32_t i = n; i < owned; i++) t[i] = -1;
    }
    uint64_t b = pos;
    for (auto v : slots) if (v != -1) out_ids[pos++] = v;
    if (reverse) std::reverse(out_ids + b, out_ids + pos);
  }
  out_offs[n_sent] = pos;
  return 0;
}

}  // extern "C"
