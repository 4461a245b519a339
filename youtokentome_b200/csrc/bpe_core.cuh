// bpe_core.cuh — host/device building blocks of the BPE hot paths.
//
// Everything here is __host__ __device__ so the very same source is exercised sequentially on the
// CPU by tests/emul (a test harness, not a product path) and in parallel by the sm_90a kernels.
// Reference behaviour restated (never copied); file:line of the reference cited per function.
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define YT_HD __host__ __device__ __forceinline__
#else
#define YT_HD inline
#endif

namespace yt {

constexpr uint32_t INVALID_CP = 0x0fffffffu;  // utf8.h:9
constexpr uint32_t SPACE_CP = 9601u;          // utils.h:9 (U+2581)
constexpr uint32_t CP_LIMIT = 0x110000u;      // dense code-point tables
constexpr uint32_t NO_ID = 0xffffffffu;       // cp2id: removed / unknown char
constexpr uint32_t DEAD = 0xffffffffu;        // token slot tombstone (tail padding of a word)
constexpr uint32_t UNK_FLAG = 0x80000000u;    // encode: pseudo token of an unknown-char run

// utils.cpp:99-101 — ASCII isspace (C locale) or U+2581.
YT_HD bool is_space_cp(uint32_t c) { return c == 32u || (c - 9u) <= 4u || c == SPACE_CP; }
YT_HD bool is_space_byte(uint8_t b) { return b == 32 || (uint8_t)(b - 9) <= 4; }
YT_HD bool is_cont(uint8_t b) { return (b & 0xc0) == 0x80; }

// utf8.cpp:20-35 — sequence length announced by a lead byte (0 = not a lead byte).
YT_HD uint32_t lead_len(uint8_t b) {
  if (b < 0x80) return 1;
  if ((b & 0xe0) == 0xc0) return 2;
  if ((b & 0xf0) == 0xe0) return 3;
  if ((b & 0xf8) == 0xf0) return 4;
  return 0;
}
YT_HD bool valid_cp(uint32_t x) { return x < 0xd800u || (x > 0xdfffu && x < 0x110000u); }  // utf8.cpp:16-18

// utf8.cpp:37-74 — decode the unit starting at s[p] (p must be a unit start); at most n-p bytes
// belong to the text.  Invalid => INVALID_CP with *len = 1.
YT_HD uint32_t decode_unit(const uint8_t *s, uint64_t p, uint64_t n, uint32_t *len) {
  uint8_t b0 = s[p];
  *len = 1;
  if (b0 < 0x80) return b0;
  uint32_t L = lead_len(b0);
  uint64_t left = n - p;
  if (L == 2 && left >= 2 && is_cont(s[p + 1])) {
    uint32_t cp = ((b0 & 0x1fu) << 6) | (s[p + 1] & 0x3fu);
    if (cp >= 0x80u && valid_cp(cp)) { *len = 2; return cp; }
  } else if (L == 3 && left >= 3 && is_cont(s[p + 1]) && is_cont(s[p + 2])) {
    uint32_t cp = ((b0 & 0x0fu) << 12) | ((s[p + 1] & 0x3fu) << 6) | (s[p + 2] & 0x3fu);
    if (cp >= 0x800u && valid_cp(cp)) { *len = 3; return cp; }
  } else if (L == 4 && left >= 4 && is_cont(s[p + 1]) && is_cont(s[p + 2]) && is_cont(s[p + 3])) {
    uint32_t cp = ((b0 & 0x07u) << 18) | ((s[p + 1] & 0x3fu) << 12) | ((s[p + 2] & 0x3fu) << 6) | (s[p + 3] & 0x3fu);
    if (cp >= 0x10000u && valid_cp(cp)) { *len = 4; return cp; }
  }
  return INVALID_CP;
}

// Is byte p the first byte of a decode unit?  The reference decodes serially (UTF8Iterator,
// utf8.h:21-64: valid sequence => advance len, else advance 1).  That recurrence is local:
// a non-continuation byte always starts a unit (it can never be consumed as a continuation);
// a continuation byte is consumed iff the nearest non-continuation byte q within 3 bytes
// before it starts a VALID sequence that covers p; otherwise it is its own (invalid) unit.
// `lo` is the first byte of the text (sequences never start before it).
YT_HD bool is_unit_start(const uint8_t *s, uint64_t p, uint64_t lo, uint64_t n) {
  if (!is_cont(s[p])) return true;
  for (uint32_t d = 1; d <= 3; d++) {
    if (p < lo + d) return true;
    uint64_t q = p - d;
    if (is_cont(s[q])) continue;
    uint32_t len;
    decode_unit(s, q, n, &len);
    return !(q + len > p);
  }
  return true;
}

// A "space unit" is an ASCII space byte or the 3 bytes E2 96 81 (U+2581).  Both always sit on
// unit starts, so word boundaries can be found on raw bytes.
YT_HD bool space_at(const uint8_t *s, uint64_t p, uint64_t n, uint32_t *len) {
  uint8_t b = s[p];
  if (is_space_byte(b)) { *len = 1; return true; }
  if (b == 0xe2 && p + 2 < n && s[p + 1] == 0x96 && s[p + 2] == 0x81) { *len = 3; return true; }
  *len = 1;
  return false;
}
// Does a space unit END right before p (or is p the start of the text)?
YT_HD bool space_before(const uint8_t *s, uint64_t p, uint64_t lo) {
  if (p == lo) return true;
  if (is_space_byte(s[p - 1])) return true;
  return p >= lo + 3 && s[p - 3] == 0xe2 && s[p - 2] == 0x96 && s[p - 1] == 0x81;
}
// Byte p starts a word (a maximal run of non-space units; compute_word_count bpe.cpp:388-418).
YT_HD bool word_start_at(const uint8_t *s, uint64_t p, uint64_t lo, uint64_t n) {
  uint32_t l;
  if (is_cont(s[p])) {
    // a continuation byte can start a word only as a stray (invalid) unit right after a space
    if (!space_before(s, p, lo)) return false;
    return true;
  }
  if (space_at(s, p, n, &l)) return false;
  return space_before(s, p, lo);
}

YT_HD uint64_t mix64(uint64_t h) {
  h ^= h >> 33; h *= 0xff51afd7ed558ccdULL; h ^= h >> 33; h *= 0xc4ceb9fe1a85ec53ULL; h ^= h >> 33;
  return h;
}
YT_HD uint64_t pair_key(uint32_t a, uint32_t b) { return ((uint64_t)a << 32) | b; }  // int2comb bpe.cpp:96-98
// Hash of a token pair for the (small, L2-resident) rule table of the encoder.  Token ids are small
// consecutive integers, so the mix must be strong: a cheap linear 32-bit hash (tried: a*K1 + b*K2)
// clusters under linear probing and cost more probes than it saved instructions (3.8 -> 4.9 ms).
YT_HD uint32_t rule_hash(uint32_t a, uint32_t b) { return (uint32_t)mix64(pair_key(a, b)); }

// Total order of MergeCandidate::operator< (bpe.cpp:110-126) as a sortable word: among equal
// counts prefer smaller max(x,y), then smaller min(x,y), then larger x.  Larger value wins.
YT_HD uint64_t pair_prio(uint32_t x, uint32_t y) {
  uint32_t mx = x > y ? x : y, mn = x > y ? y : x;
  return ((uint64_t)(0xffffffffu - mx) << 32) | ((uint64_t)(0x7fffffffu - mn) << 1) | (x >= y ? 1u : 0u);
}

// Pair multiset of a token sequence under the run rule: a run a^L contributes floor(L/2) pairs
// (a,a) (pairsInSeg bpe.cpp:140-143, build_linked_list :465-475) and each run boundary one
// cross pair.  Stops at the first DEAD slot.  emit(key, multiplicity).
template <class Emit>
YT_HD void for_each_pair(const uint32_t *t, uint32_t cap, Emit emit) {
  uint32_t i = 0;
  if (cap == 0) return;
  uint32_t a = t[0];
  if (a == DEAD) return;
  while (true) {
    uint32_t j = i + 1, b = DEAD;
    while (j < cap && (b = t[j]) == a) j++;
    if (j >= cap) b = DEAD;
    uint32_t run = j - i;
    if (run >= 2) emit(pair_key(a, a), (uint64_t)(run >> 1));
    if (b == DEAD) return;
    emit(pair_key(a, b), (uint64_t)1);
    i = j; a = b;
  }
}

// Number of live tokens of a word slot range.
YT_HD uint32_t live_len(const uint32_t *t, uint32_t cap) {
  uint32_t n = 0;
  while (n < cap && t[n] != DEAD) n++;
  return n;
}

// Does the word contain x immediately followed by y?
YT_HD bool has_pair(const uint32_t *t, uint32_t cap, uint32_t x, uint32_t y) {
  if (cap < 2) return false;
  uint32_t a = t[0];
  for (uint32_t i = 1; i < cap; i++) {
    uint32_t b = t[i];
    if (b == DEAD) return false;
    if (a == x && b == y) return true;
    a = b;
  }
  return false;
}

// Greedy left-to-right, non-overlapping rewrite x y -> z in place (stress_test.cpp:181-188;
// for x == y a run x^L becomes z^(L/2) + x^(L%2), bpe.cpp:654-690).  The freed tail is padded
// with DEAD.  Returns the number of merges.
YT_HD uint32_t rewrite_word(uint32_t *t, uint32_t cap, uint32_t x, uint32_t y, uint32_t z) {
  uint32_t r = 0, w = 0, merges = 0;
  while (r < cap) {
    uint32_t a = t[r];
    if (a == DEAD) break;
    if (a == x && r + 1 < cap && t[r + 1] == y) { t[w++] = z; r += 2; merges++; }
    else { t[w++] = a; r++; }
  }
  for (uint32_t k = w; k < r; k++) t[k] = DEAD;
  return merges;
}

// ---------------------------------------------------------------------------------------------
// Philox4x32-10 — BPE-dropout draws (replaces the reference's global std::mt19937, bpe.cpp:1415).
// ---------------------------------------------------------------------------------------------
YT_HD uint32_t mulhi32(uint32_t a, uint32_t b) { return (uint32_t)(((uint64_t)a * b) >> 32); }
YT_HD uint32_t philox_first(uint32_t k0, uint32_t k1, uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3) {
  for (int r = 0; r < 10; r++) {
    uint32_t n0 = mulhi32(0xCD9E8D57u, c2) ^ c1 ^ k0, n1 = 0xCD9E8D57u * c2;
    uint32_t n2 = mulhi32(0xD2511F53u, c0) ^ c3 ^ k1, n3 = 0xD2511F53u * c0;
    c0 = n0; c1 = n1; c2 = n2; c3 = n3;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  return c0;
}
// One Bernoulli draw of DropoutQueue::pop (bpe.cpp:1440): true = skip this candidate.
// counter = (sentence index, byte offset of the word inside the sentence, draw number).
YT_HD bool dropout_skip(uint64_t seed, uint64_t sent, uint32_t word_off, uint32_t draw, uint64_t thresh) {
  uint32_t r = philox_first((uint32_t)seed, (uint32_t)(seed >> 32), (uint32_t)sent, (uint32_t)(sent >> 32), word_off, draw);
  return (uint64_t)r < thresh;
}


// ---------------------------------------------------------------------------------------------
// encode one word (the body of encode_sentence's per-word loop, bpe.cpp:1505-1614):
// bytes [p0, end of the non-space byte run) of a sentence [lo, hi) -> tokens written to t[0..n).
// t and r are private arrays with (run bytes + 1) entries.  Unknown-char runs collapse to one
// pseudo token (UNK_FLAG) that never merges; invalid units vanish (decode_utf8 utf8.cpp:111-128).
// Merges: minimum rule index, leftmost first (MergeEvent2::operator< bpe.cpp:1475-1478).
// rank(a, b, &z) returns the rule index of (a,b) or NO_RANK_V.  zr (optional, same size as r) caches the z
// of every cached rank so a merge needs no second probe.  Returns n (0 = no word);
// *slots_owned = entries of t that belong to this word.
//
// BPE-dropout (drop_thresh > 0) models the reference's DropoutQueue exactly (bpe.cpp:1417-1453
// + the caller's loop :1560-1589): the queue holds one event (rule, position) per adjacent
// pair that has a rule, PLUS the stale events of pairs a merge destroyed (they stay queued until
// a pop accepts them and the caller discards them, :1569-1572).  One pop() walks the events in
// (rule, position) order and draws once per event; the first event that is not skipped is
// returned, the skipped ones are re-queued; if every event is skipped the word is finished.
// Valid events are implicit (r[i] of live node i); stale ones are kept in st_rule/st_pos.
// aux = 6 * (run bytes + 1) extra uint32 of private scratch (only read when drop_thresh > 0).
// ---------------------------------------------------------------------------------------------
constexpr uint32_t NO_RANK_V = 0xffffffffu;

// A quirk of the reference, reproduced: encode_sentence starts a word's output at the first node whose token id is
// not 0, because merged-away nodes carry id 0 (bpe.cpp:1591-1596).  When U+2581 itself has id 0 — no special token
// sits at 0, e.g. pad_id = -1 — a word-initial "▁" that no rule merged is therefore dropped from the output.
YT_HD uint32_t drop_unmerged_space0(int32_t *t, uint32_t n, uint32_t space_id) {
  if (space_id != 0 || n == 0 || t[0] != 0) return n;
  for (uint32_t i = 0; i + 1 < n; i++) t[i] = t[i + 1];
  return n - 1;
}

template <class RankFn>
YT_HD uint32_t encode_word(const uint8_t *s, uint64_t p0, uint64_t lo, uint64_t hi, const uint32_t *cp2id,
                           uint32_t space_id, RankFn rank, uint32_t *zr, uint64_t drop_thresh, uint64_t seed, uint64_t sent_index,
                           int32_t *t, uint32_t *r, uint32_t *aux, uint32_t *slots_owned) {
  uint32_t n = 1, l;
  bool last_unk = false;
  uint64_t q = p0;
  while (q < hi && !space_at(s, q, hi, &l)) {
    uint32_t cp = decode_unit(s, q, hi, &l);
    q += l;
    if (cp == INVALID_CP) continue;
    uint32_t id = cp2id[cp];
    if (id == NO_ID) {
      if (!last_unk) t[n++] = (int32_t)(UNK_FLAG | 1u);
      last_unk = true;
    } else { t[n++] = (int32_t)id; last_unk = false; }
  }
  const uint32_t owned = (uint32_t)(q - p0) + 1;
  *slots_owned = owned;
  if (n == 1) return 0;  // no valid unit: the reference sees no word
  t[0] = (int32_t)space_id;
  uint32_t z = 0;
  for (uint32_t i = 0; i + 1 < n; i++) { r[i] = rank((uint32_t)t[i], (uint32_t)t[i + 1], &z); if (zr) zr[i] = z; }
  if (drop_thresh == 0) {
    while (n > 1) {
      uint32_t best = NO_RANK_V, bi = 0;
      for (uint32_t i = 0; i + 1 < n; i++)
        if (r[i] < best) { best = r[i]; bi = i; }
      if (best == NO_RANK_V) break;
      if (zr) z = zr[bi]; else rank((uint32_t)t[bi], (uint32_t)t[bi + 1], &z);
      t[bi] = (int32_t)z;
      for (uint32_t i = bi + 1; i + 1 < n; i++) { t[i] = t[i + 1]; if (i + 2 < n) { r[i] = r[i + 1]; if (zr) zr[i] = zr[i + 1]; } }
      n--;
      if (bi > 0) { r[bi - 1] = rank((uint32_t)t[bi - 1], (uint32_t)t[bi], &z); if (zr) zr[bi - 1] = z; }
      if (bi + 1 < n) { r[bi] = rank((uint32_t)t[bi], (uint32_t)t[bi + 1], &z); if (zr) zr[bi] = z; }
    }
    return drop_unmerged_space0(t, n, space_id);
  }
  // ---- dropout: stable node positions (linked list) + explicit stale events
  const uint32_t NIL = 0xffffffffu;
  uint32_t *nx = aux, *pv = aux + owned, *st_rule = aux + 2 * owned, *st_pos = aux + 4 * owned;
  for (uint32_t i = 0; i < n; i++) { nx[i] = i + 1 < n ? i + 1 : NIL; pv[i] = i ? i - 1 : NIL; }
  r[n - 1] = NO_RANK_V;
  uint32_t n_stale = 0, draw = 0, live = n;
  const uint32_t word_off = (uint32_t)(p0 - lo);
  while (true) {
    // one pop(): visit events in increasing (rule, pos); lr/lp = last visited key
    uint32_t lr = 0, lp = 0, br = NO_RANK_V, bp = 0, bstale = NIL;
    bool have_last = false, accepted = false;
    while (true) {
      br = NO_RANK_V; bstale = NIL;
      for (uint32_t i = 0; i != NIL; i = nx[i]) {  // valid events (node 0 is always alive)
        uint32_t ri = r[i];
        if (ri == NO_RANK_V) continue;
        if (have_last && (ri < lr || (ri == lr && i <= lp))) continue;
        if (ri < br || (ri == br && i < bp)) { br = ri; bp = i; }
      }
      for (uint32_t k = 0; k < n_stale; k++) {
        uint32_t ri = st_rule[k], pi = st_pos[k];
        if (have_last && (ri < lr || (ri == lr && pi <= lp))) continue;
        if (ri < br || (ri == br && pi < bp)) { br = ri; bp = pi; bstale = k; }
      }
      if (br == NO_RANK_V) break;                                                     // queue exhausted
      if (!dropout_skip(seed, sent_index, word_off, draw++, drop_thresh)) { accepted = true; break; }
      lr = br; lp = bp; have_last = true;                                             // skipped
    }
    if (!accepted) break;  // every event skipped (or none left): word finished (bpe.cpp:1430-1436)
    if (bstale != NIL) {   // a stale event was popped: the caller drops it (bpe.cpp:1569-1572)
      n_stale--;
      st_rule[bstale] = st_rule[n_stale]; st_pos[bstale] = st_pos[n_stale];
      continue;
    }
    const uint32_t p1 = bp, p2 = nx[p1], pl = pv[p1], p3 = nx[p2];
    if (pl != NIL && r[pl] != NO_RANK_V) { st_rule[n_stale] = r[pl]; st_pos[n_stale++] = pl; }
    if (r[p2] != NO_RANK_V) { st_rule[n_stale] = r[p2]; st_pos[n_stale++] = p2; }
    rank((uint32_t)t[p1], (uint32_t)t[p2], &z);
    t[p1] = (int32_t)z;
    nx[p1] = p3;
    if (p3 != NIL) pv[p3] = p1;
    r[p2] = NO_RANK_V;
    live--;
    if (pl != NIL) r[pl] = rank((uint32_t)t[pl], (uint32_t)t[p1], &z);
    r[p1] = p3 != NIL ? rank((uint32_t)t[p1], (uint32_t)t[p3], &z) : NO_RANK_V;
  }
  // compact the live nodes to the front of t (ascending positions, so writes trail reads)
  uint32_t w = 0;
  for (uint32_t i = 0; i != NIL; i = nx[i]) t[w++] = t[i];
  return drop_unmerged_space0(t, live, space_id);
}

}  // namespace yt
