// oracle/replay_rng.h — TEST INFRASTRUCTURE ONLY (never part of the product).
//
// Force-included (-include) ahead of the unmodified reference sources by oracle/Makefile for
// _ref/libyttm_ref_replay.so.  The reference draws BPE-dropout decisions from one global
// `std::mt19937 rnd` (bpe.cpp:1415) through `uniform_real_distribution<>(0, 1)`; the macro at the
// bottom turns that declaration into a `std::yttm_replay_engine`, whose words are the product's
// Philox4x32-10 draws (youtokentome_b200/csrc/bpe_core.cuh: dropout_skip).
//
// libstdc++'s uniform_real_distribution<double>(0, 1) takes two words of a 32-bit engine per
// draw, low word first: u = (g1 + g2 * 2^32) / 2^64.  The engine answers 0 and then r, the first
// output word of Philox4x32-10 with counter (sentence lo, sentence hi, word byte offset, draw)
// and key (seed lo, seed hi), so u = r / 2^32 exactly and the reference skips an event iff
// r / 2^32 < p.  Every r advances the draw number.
//
// The key is per thread: oracle/ref_replay.cpp sets it before encoding one word.
#pragma once
#include <cstdint>
#include <random>

namespace yttm_replay {
struct Key {
  uint64_t seed = 0, sent = 0;
  uint32_t word_off = 0, draw = 0;
  uint64_t calls = 0;  // engine words handed out since set_key (two per draw)
};
inline Key &key() {
  static thread_local Key k;
  return k;
}
inline void set_key(uint64_t seed, uint64_t sent, uint32_t word_off) {
  Key &k = key();
  k.seed = seed; k.sent = sent; k.word_off = word_off; k.draw = 0; k.calls = 0;
}
// Philox4x32-10 (Salmon et al., SC'11), first output word.
inline uint32_t philox_first(uint32_t k0, uint32_t k1, uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3) {
  for (int r = 0; r < 10; r++) {
    const uint64_t p0 = (uint64_t)0xD2511F53u * c0, p1 = (uint64_t)0xCD9E8D57u * c2;
    const uint32_t n0 = (uint32_t)(p1 >> 32) ^ c1 ^ k0, n1 = (uint32_t)p1;
    const uint32_t n2 = (uint32_t)(p0 >> 32) ^ c3 ^ k1, n3 = (uint32_t)p0;
    c0 = n0; c1 = n1; c2 = n2; c3 = n3;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  return c0;
}
}  // namespace yttm_replay

namespace std {
struct yttm_replay_engine {
  typedef uint32_t result_type;
  static constexpr result_type min() { return 0; }
  static constexpr result_type max() { return 0xffffffffu; }
  yttm_replay_engine() {}
  explicit yttm_replay_engine(result_type) {}
  void seed(result_type = 0) {}
  result_type operator()() {
    yttm_replay::Key &k = yttm_replay::key();
    if (k.calls++ % 2 == 0) return 0;  // the low word of the canonical draw
    return yttm_replay::philox_first((uint32_t)k.seed, (uint32_t)(k.seed >> 32), (uint32_t)k.sent,
                                     (uint32_t)(k.sent >> 32), k.word_off, k.draw++);
  }
};
}  // namespace std

#define mt19937 yttm_replay_engine
