// train.cu — hot path (a): BPE training on one H100.
//
// Replaces, behind the C ABI of include/yttm_b200.h, the data-parallel phases of the
// reference's learn_bpe_from_string (youtokentome/cpp/bpe.cpp:859-1293):
//   char_hist_kernel     <- compute_char_count            (bpe.cpp:839-857, utf8.cpp:37-74)
//   word_insert_kernel   <- compute_word_count / VectorSegment (bpe.cpp:28-54, 388-418)
//   word_len/tokenise    <- remove_rare_chars + tokenisation   (bpe.cpp:357-380, 405-411)
//   pair_hist_kernel     <- build_linked_list pair2cnt     (bpe.cpp:436-478)
//   merge_loop_kernel    <- main loop + worker_doing_merge + PriorityQueue
//                           (bpe.cpp:1121-1282, 601-811, 149-314; order :110-126)
// Design (GPU-first, not a port): words are deduplicated on the device, their tokens live in
// one packed uint32 buffer (offsets + uint64 frequencies beside it) that stays resident in
// HBM/L2; the whole merge loop runs inside ONE persistent cooperative kernel (grid-wide
// barriers instead of the reference's mutex/condvar ping-pong): each iteration is an exact
// arg-max over a device open-addressed pair->count table followed by a scan of the packed
// tokens that rewrites the affected words in place and patches the table with atomics.
#include <cooperative_groups.h>

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <unistd.h>

#include "common.cuh"

namespace cg = cooperative_groups;
using namespace yt;

namespace {

constexpr unsigned long long PK_EMPTY = 0xFFFFFFFFFFFFFFFFull;
constexpr uint64_t POS_MASK = (1ull << 40) - 1;

// ------------------------------------------------------------------------------------------
// pair -> count table: open addressing, linear probing, SoA (keys / counts) so the arg-max
// sweep streams 8 B per slot and touches keys only for candidates.  The table is cut into
// `nparts` PARTITIONS of R = rmask + 1 slots (R a power of two): a key lives in partition
// mulhi(hash_hi, nparts) and probes inside it (wrapping at the partition's end).  Inside the merge
// loop partition b belongs to block b alone (merge_loop.cuh); the one-off histogram kernels below
// write it from everywhere with atomics.
// ------------------------------------------------------------------------------------------
struct PairTab {
  unsigned long long *keys;
  unsigned long long *cnts;
  uint32_t rmask;      // slots per partition - 1
  uint32_t nparts;
  uint32_t *n_keys;    // occupied slots (keys never leave between rebuilds)
  uint32_t *overflow;  // a partition ran full: the update was dropped, the host rebuilds a larger table
};
__device__ __forceinline__ uint64_t tab_slots(const PairTab &t) { return (uint64_t)t.nparts * ((uint64_t)t.rmask + 1); }
__device__ __forceinline__ uint32_t pair_part(const PairTab &t, uint64_t h) { return mulhi32((uint32_t)(h >> 32), t.nparts); }

// Add delta to `key` inside the partition that starts at slot `base`, first probe at base + i0.
// Returns true when the key was inserted.  A full partition drops the update and raises the flag.
template <bool CAS_FIRST = false>
__device__ __forceinline__ bool pair_add_at(const PairTab &t, uint64_t base, uint32_t i0, uint64_t key, long long delta,
                                            uint64_t *slot_out = nullptr) {
  for (uint32_t probe = 0; probe <= t.rmask; probe++) {
    const uint64_t h = base + ((i0 + probe) & t.rmask);
    unsigned long long k;
    bool fresh = false;
    if (CAS_FIRST) {  // a pair that most likely is new: claim without looking
      k = atomicCAS(t.keys + h, PK_EMPTY, (unsigned long long)key);
      if (k == PK_EMPTY) { fresh = true; k = key; }
    } else {
      k = __ldcg(t.keys + h);
#ifdef YT_SIMT_EMU
      emu::yield();  // test harness: other fibers run between the load and the CAS, so the lost-race path is exercised
#endif
      if (k == PK_EMPTY) {
        k = atomicCAS(t.keys + h, PK_EMPTY, (unsigned long long)key);
        if (k == PK_EMPTY) { fresh = true; k = key; }
      }
    }
    if (k == key) {
      atomicAdd(t.cnts + h, (unsigned long long)delta);
      if (fresh) atomicAdd(t.n_keys, 1u);
      if (slot_out) *slot_out = h;
      return fresh;
    }
  }
  atomicExch(t.overflow, 1u);
  return false;
}
__device__ __forceinline__ void pair_add(const PairTab &t, uint64_t key, long long delta) {
  const uint64_t h = mix64(key);
  pair_add_at(t, (uint64_t)pair_part(t, h) * ((uint64_t)t.rmask + 1), (uint32_t)h & t.rmask, key, delta);
}

// ------------------------------------------------------------------------------------------
// phase 1: decode units + code point histogram
// ------------------------------------------------------------------------------------------
constexpr int HIST_SMEM_BINS = 2048;  // every 1- and 2-byte code point

// decode_unit (bpe_core.cuh) on four bytes held in a register (b0 in the low byte): bytes beyond the text are spaces
// there, which end every sequence exactly like the bounds check of the byte-wise version (a space is no continuation).
__device__ __forceinline__ uint32_t decode_reg(uint32_t w, uint32_t *len) {
  const uint32_t b0 = w & 0xffu, b1 = (w >> 8) & 0xffu, b2 = (w >> 16) & 0xffu, b3 = w >> 24;
  *len = 1;
  if (b0 < 0x80u) return b0;
  const bool c1 = (b1 & 0xc0u) == 0x80u, c2 = (b2 & 0xc0u) == 0x80u, c3 = (b3 & 0xc0u) == 0x80u;
  if ((b0 & 0xe0u) == 0xc0u) {
    const uint32_t cp = ((b0 & 0x1fu) << 6) | (b1 & 0x3fu);
    if (c1 && cp >= 0x80u) { *len = 2; return cp; }
  } else if ((b0 & 0xf0u) == 0xe0u) {
    const uint32_t cp = ((b0 & 0x0fu) << 12) | ((b1 & 0x3fu) << 6) | (b2 & 0x3fu);
    if (c1 && c2 && cp >= 0x800u && valid_cp(cp)) { *len = 3; return cp; }
  } else if ((b0 & 0xf8u) == 0xf0u) {
    const uint32_t cp = ((b0 & 0x07u) << 18) | ((b1 & 0x3fu) << 12) | ((b2 & 0x3fu) << 6) | (b3 & 0x3fu);
    if (c1 && c2 && c3 && cp >= 0x10000u && valid_cp(cp)) { *len = 4; return cp; }
  }
  return INVALID_CP;
}
__device__ __forceinline__ uint32_t funnel_r(uint32_t lo, uint32_t hi, uint32_t shift_bits) {
  return shift_bits ? (lo >> shift_bits) | (hi << (32u - shift_bits)) : lo;
}
// the aligned 32-bit word at text position p (p + address alignment is a multiple of 4), spaces outside [0, n)
__device__ __forceinline__ uint32_t text_word(const uint8_t *__restrict__ s, int64_t p, int64_t n) {
  if (p >= 0 && p + 4 <= n) return *reinterpret_cast<const uint32_t *>(s + p);
  uint32_t w = 0x20202020u;
  for (int k = 0; k < 4; k++)
    if (p + k >= 0 && p + k < n) w = (w & ~(0xffu << (8 * k))) | ((uint32_t)s[p + k] << (8 * k));
  return w;
}

// Phase 1 with 16 bytes per thread: one aligned 16-byte load, the 4 bytes before and after come from the neighbour
// lanes by shuffle, and unit starts / code points are decided on that 24-byte register window (is_unit_start and
// decode_unit restated on registers: a continuation byte is consumed iff the nearest non-continuation byte within 3
// before it starts a valid sequence that covers it).  Round 1 issued 3 - 8 byte loads per position (57 GB/s).
__global__ void __launch_bounds__(512) char_hist_kernel(const uint8_t *__restrict__ s, uint64_t n_text,
                                                        unsigned long long *__restrict__ hist) {
  __shared__ uint32_t sh[HIST_SMEM_BINS];
  __shared__ unsigned long long s_units;
  for (int i = threadIdx.x; i < HIST_SMEM_BINS; i += blockDim.x) sh[i] = 0;
  if (threadIdx.x == 0) s_units = 0;
  __syncthreads();
  const int64_t n = (int64_t)n_text;
  const int64_t mis = (int64_t)(reinterpret_cast<uintptr_t>(s) & 15u);  // text position -mis is 16-byte aligned
  const int64_t n_vec = (n + mis + 15) / 16;
  const unsigned lane = threadIdx.x & 31;
  uint64_t units = 0;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int64_t rounds = (n_vec + stride - 1) / stride;
  for (int64_t r = 0; r < rounds; r++) {  // warp-uniform trip count: every lane takes part in the shuffles
    const int64_t v = r * stride + (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t p0 = v * 16 - mis;
    uint32_t w[6];
    if (v < n_vec && p0 >= 0 && p0 + 16 <= n) {
      const uint4 q = *reinterpret_cast<const uint4 *>(s + p0);
      w[1] = q.x; w[2] = q.y; w[3] = q.z; w[4] = q.w;
    } else {
#pragma unroll
      for (int k = 0; k < 4; k++) w[1 + k] = v < n_vec ? text_word(s, p0 + 4 * k, n) : 0x20202020u;
    }
    w[0] = __shfl_up_sync(0xffffffffu, w[4], 1);
    w[5] = __shfl_down_sync(0xffffffffu, w[1], 1);
    if (lane == 0) w[0] = text_word(s, p0 - 4, n);
    if (lane == 31) w[5] = text_word(s, p0 + 16, n);
    if (v >= n_vec) continue;
#pragma unroll
    for (int i = 0; i < 16; i++) {
      const int64_t p = p0 + i;
      const int j = i + 4;  // window index of the byte
      const uint32_t four = funnel_r(w[j >> 2], w[(j >> 2) + 1 < 6 ? (j >> 2) + 1 : 5], (uint32_t)(j & 3) * 8u);
      const uint32_t b = four & 0xffu;
      bool start = true;
      if ((b & 0xc0u) == 0x80u) {  // continuation byte: covered by a valid sequence that starts 1..3 bytes earlier?
#pragma unroll
        for (int d = 1; d <= 3; d++) {
          const int jq = j - d;
          const uint32_t fq = funnel_r(w[jq >> 2], w[(jq >> 2) + 1], (uint32_t)(jq & 3) * 8u);
          if ((fq & 0xc0u) != 0x80u) {
            uint32_t lq;
            decode_reg(fq, &lq);
            start = !(lq > (uint32_t)d);
            break;
          }
        }
      }
      if (!start || p < 0 || p >= n) continue;
      units++;
      uint32_t len;
      const uint32_t cp = decode_reg(four, &len);
      if (cp == INVALID_CP || is_space_cp(cp)) continue;
      if (cp < HIST_SMEM_BINS) atomicAdd(&sh[cp], 1u);
      else atomicAdd(hist + cp, 1ull);
    }
  }
  for (int o = 16; o > 0; o >>= 1) units += __shfl_xor_sync(0xffffffffu, units, o);
  if ((threadIdx.x & 31) == 0 && units) atomicAdd(&s_units, (unsigned long long)units);
  __syncthreads();
  for (int i = threadIdx.x; i < HIST_SMEM_BINS; i += blockDim.x)
    if (sh[i]) atomicAdd(hist + i, (unsigned long long)sh[i]);
  if (threadIdx.x == 0 && s_units) atomicAdd(hist + CP_LIMIT, s_units);
}

// ------------------------------------------------------------------------------------------
// phase 2: word split + dedup.  Key word = ((tag24 << 40) | (byte position + 1)) of the first
// occurrence that claimed the slot; duplicates are verified byte by byte against it.
// ------------------------------------------------------------------------------------------
struct WordTab {
  unsigned long long *keys;  // 0 = empty
  unsigned long long *cnts;
  uint64_t mask;
};
// counters: [0] word occurrences, [1] unique words, [2] overflow flag, [3] compaction cursor

__device__ __forceinline__ bool same_word(const uint8_t *s, uint64_t n, uint64_t a, uint64_t b, uint64_t len) {
  if (a + len > n) return false;
  for (uint64_t i = 0; i < len; i++)
    if (s[a + i] != s[b + i]) return false;
  uint32_t l;
  return a + len == n || space_at(s, a + len, n, &l);
}

// The word table's hash of the word that starts at byte p: FNV-1a over its bytes, then mixed with its length.  It does
// not depend on where the word lies, so a word hashes alike in a piece of the corpus and in the word arena.
__device__ __forceinline__ uint64_t word_hash(const uint8_t *__restrict__ s, uint64_t n, uint64_t p, uint64_t *len_out) {
  uint64_t h = 0xcbf29ce484222325ull, q = p;
  uint32_t l;
  while (q < n && !space_at(s, q, n, &l)) { h = (h ^ s[q]) * 0x100000001b3ull; q++; }
  *len_out = q - p;
  return mix64(h ^ ((q - p) << 1));
}

// insert the word that starts at byte p (weight = its number of occurrences) ; returns false when the table is full
__device__ __forceinline__ bool word_table_insert(const uint8_t *__restrict__ s, uint64_t n, uint64_t p, const WordTab &wt,
                                                  unsigned long long *counters, uint64_t max_unique,
                                                  unsigned long long weight) {
  uint64_t len;
  const uint64_t h = word_hash(s, n, p, &len);
  uint64_t tag = h >> 40;
  unsigned long long mine = (tag << 40) | (p + 1);
  uint64_t slot = h & wt.mask;
  for (uint64_t probe = 0; probe <= wt.mask; probe++) {
    unsigned long long k = __ldcg(wt.keys + slot);
    if (k == 0) {
      if (__ldcg(counters + 1) >= max_unique) { atomicExch(counters + 2, 1ull); return false; }
      k = atomicCAS(wt.keys + slot, 0ull, mine);
      if (k == 0) { atomicAdd(counters + 1, 1ull); atomicAdd(wt.cnts + slot, weight); return true; }
    }
    if ((k >> 40) == tag && same_word(s, n, (k & POS_MASK) - 1, p, len)) { atomicAdd(wt.cnts + slot, weight); return true; }
    slot = (slot + 1) & wt.mask;
  }
  return false;
}

// Word split + dedup of running text: thread per byte position; a position that starts a word hashes it and inserts
// it into the global word table (exact byte compare on a tag match).  Instruction
// bound — the per-word hash / compare loops run with ~5 of 32 lanes active.  A variant that first aggregated the words
// of a 64 KB chunk in a shared-memory table (to take the hot words' same-address atomics off L2) was measured SLOWER
// (more warp instructions than the atomics it saved) and was dropped.
__global__ void __launch_bounds__(256) word_insert_kernel(const uint8_t *__restrict__ s, uint64_t n, uint64_t lo, uint64_t hi,
                                                          WordTab wt, unsigned long long *counters, uint64_t max_unique) {
  uint64_t stride = (uint64_t)gridDim.x * blockDim.x;   // word starts in [lo, hi) of the text [0, n)
  uint64_t occ = 0;
  for (uint64_t p = lo + (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; p < hi; p += stride) {
    if (!word_start_at(s, p, 0, n)) continue;
    occ++;
    word_table_insert(s, n, p, wt, counters, max_unique, 1ull);
  }
  for (int o = 16; o > 0; o >>= 1) occ += __shfl_xor_sync(0xffffffffu, occ, o);
  if ((threadIdx.x & 31) == 0 && occ) atomicAdd(counters + 0, (unsigned long long)occ);
}

// Multi-GPU import: the "text" is a list of words (word i starts at byte base + pos[i], a space follows it) that other
// ranks found freq[i] times each (yttm_train_dist_export_words); same table, same exact byte compare.
__global__ void __launch_bounds__(256) word_insert_list_kernel(const uint8_t *__restrict__ s, uint64_t n, uint64_t base,
                                                               const uint64_t *__restrict__ pos,
                                                               const uint64_t *__restrict__ freq, uint64_t n_list,
                                                               WordTab wt, unsigned long long *counters, uint64_t max_unique) {
  uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  unsigned long long occ = 0;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_list; i += stride) {
    occ += freq[i];
    word_table_insert(s, n, base + pos[i], wt, counters, max_unique, (unsigned long long)freq[i]);
  }
  for (int o = 16; o > 0; o >>= 1) occ += __shfl_xor_sync(0xffffffffu, occ, o);
  if ((threadIdx.x & 31) == 0 && occ) atomicAdd(counters + 0, occ);
}

// Multi-GPU export: unique word w of this rank goes to rank owner(w) = hash(bytes) % world (every rank uses the same
// function, so equal words meet on one rank).  PASS 0 counts bytes (word + one space) and words per destination;
// PASS 1 writes them behind the per-destination cursors (any order inside a destination).
template <int PASS>
__global__ void __launch_bounds__(256) word_export_kernel(const uint8_t *__restrict__ s, uint64_t n,
                                                          const uint64_t *__restrict__ wpos,
                                                          const uint64_t *__restrict__ wfreq, uint64_t n_unique,
                                                          uint32_t world, unsigned long long *cur_bytes /* [world] */,
                                                          unsigned long long *cur_words /* [world] */,
                                                          const unsigned long long *byte_base /* [world], PASS 1 */,
                                                          uint8_t *__restrict__ out_bytes, uint64_t *__restrict__ out_pos,
                                                          uint64_t *__restrict__ out_freq) {
  uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  for (uint64_t w = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; w < n_unique; w += stride) {
    const uint64_t p = wpos[w];
    uint64_t h = 0xcbf29ce484222325ull, q = p;
    uint32_t l;
    while (q < n && !space_at(s, q, n, &l)) { h = (h ^ s[q]) * 0x100000001b3ull; q++; }
    const uint64_t len = q - p;
    const uint32_t dst = mulhi32((uint32_t)(mix64(h + len) >> 32), world);
    const unsigned long long at = atomicAdd(cur_bytes + dst, (unsigned long long)(len + 1));
    const unsigned long long idx = atomicAdd(cur_words + dst, 1ull);
    if (PASS == 1) {
      for (uint64_t i = 0; i < len; i++) out_bytes[at + i] = s[p + i];
      out_bytes[at + len] = ' ';
      out_pos[idx] = at - byte_base[dst];  // relative to the destination's first byte
      out_freq[idx] = wfreq[w];
    }
  }
}

__global__ void word_compact_kernel(WordTab wt, unsigned long long *counters, uint64_t *__restrict__ wpos,
                                    uint64_t *__restrict__ wfreq) {
  uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i <= wt.mask; i += stride) {
    unsigned long long k = wt.keys[i];
    if (k == 0) continue;
    unsigned long long idx = atomicAdd(counters + 3, 1ull);
    wpos[idx] = (k & POS_MASK) - 1;
    wfreq[idx] = wt.cnts[i];
  }
}

// ---- fed corpus: the distinct words of one piece (wpos / wfreq, positions in the piece) into the persistent table,
// whose keys point into the word arena `a` (alen bytes; every word there is followed by one ' ').  Two passes, so
// that no thread compares against arena bytes that another thread is still writing:
//   lookup: a word already in the table adds its count; a new word records len + 1 (its arena bytes) in mlen and is
//           counted in counters[5];
//   (the host scans mlen into arena offsets and grows the arena / the table)
//   insert: a new word copies its bytes + ' ' to the arena and claims an empty slot.  No byte compare: the new words
//           differ from each other (one per-piece table) and from every word of the table (the lookup pass).
__global__ void __launch_bounds__(256) word_merge_lookup_kernel(const uint8_t *__restrict__ s, uint64_t n,
                                                                const uint64_t *__restrict__ wpos,
                                                                const uint64_t *__restrict__ wfreq, uint64_t n_words,
                                                                WordTab ft, const uint8_t *__restrict__ a,
                                                                unsigned long long *__restrict__ mlen,
                                                                unsigned long long *counters) {
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_words; i += stride) {
    const uint64_t p = wpos[i];
    uint64_t len;
    const uint64_t h = word_hash(s, n, p, &len), tag = h >> 40;
    unsigned long long miss = len + 1;
    for (uint64_t slot = h & ft.mask;; slot = (slot + 1) & ft.mask) {   // the table is at most half full
      const unsigned long long k = ft.keys[slot];
      if (k == 0) break;
      if ((k >> 40) != tag) continue;
      const uint64_t q = (k & POS_MASK) - 1;
      uint64_t j = 0;
      while (j < len && a[q + j] == s[p + j]) j++;   // an arena word is followed by ' ', which no word byte equals
      if (j == len && a[q + len] == ' ') {
        atomicAdd(ft.cnts + slot, (unsigned long long)wfreq[i]);
        miss = 0;
        break;
      }
    }
    mlen[i] = miss;
    if (miss) atomicAdd(counters + 5, 1ull);
  }
}

__global__ void __launch_bounds__(256) word_merge_insert_kernel(const uint8_t *__restrict__ s, uint64_t n,
                                                                const uint64_t *__restrict__ wpos,
                                                                const uint64_t *__restrict__ wfreq, uint64_t n_words,
                                                                const unsigned long long *__restrict__ mlen,
                                                                const unsigned long long *__restrict__ moff,
                                                                WordTab ft, uint8_t *__restrict__ a, uint64_t alen) {
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_words; i += stride) {
    if (!mlen[i]) continue;
    const uint64_t p = wpos[i], at = alen + moff[i];
    uint64_t len;
    const uint64_t h = word_hash(s, n, p, &len);
    for (uint64_t j = 0; j < len; j++) a[at + j] = s[p + j];
    a[at + len] = ' ';
    const unsigned long long key = ((h >> 40) << 40) | (at + 1);
    uint64_t slot = h & ft.mask;
    while (atomicCAS(ft.keys + slot, 0ull, key) != 0ull) slot = (slot + 1) & ft.mask;
    ft.cnts[slot] = wfreq[i];
  }
}

// The persistent table moved to a larger one (old -> nt): every word is hashed again from its arena bytes.
__global__ void __launch_bounds__(256) word_table_rehash_kernel(WordTab old, WordTab nt, const uint8_t *__restrict__ a,
                                                                uint64_t alen) {
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i <= old.mask; i += stride) {
    const unsigned long long k = old.keys[i];
    if (k == 0) continue;
    uint64_t len;
    const uint64_t h = word_hash(a, alen, (k & POS_MASK) - 1, &len);
    uint64_t slot = h & nt.mask;
    while (atomicCAS(nt.keys + slot, 0ull, k) != 0ull) slot = (slot + 1) & nt.mask;
    nt.cnts[slot] = old.cnts[i];
  }
}

// freq x tokens of every word below 2^43 (the signed 44-bit count change of the merge loop's exchange entries, as
// yttm_train_import_words checks): a text shard cannot exceed it, a fed corpus can.  lens: tokens per word.
__global__ void word_count_limit_kernel(const unsigned long long *__restrict__ lens, const uint64_t *__restrict__ wfreq,
                                        uint64_t n_words, unsigned long long *bad) {
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  for (uint64_t w = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; w < n_words; w += stride)
    if (lens[w] && wfreq[w] >= (1ull << 43) / lens[w]) atomicExch(bad, 1ull);
}

// tokens of one unique word: [space_id] + ids of kept chars; removed / invalid units vanish.
// MODE 0: count only.  MODE 1: write.
template <int MODE>
__global__ void word_tokens_kernel(const uint8_t *__restrict__ s, uint64_t n, const uint64_t *__restrict__ wpos,
                                   uint64_t n_unique, const uint32_t *__restrict__ cp2id, uint32_t space_id,
                                   unsigned long long *__restrict__ lens, const unsigned long long *__restrict__ scan,
                                   uint32_t *__restrict__ tok, uint32_t *__restrict__ off) {
  uint64_t w = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (w >= n_unique) return;
  uint64_t q = wpos[w];
  uint32_t kept = 0, l;
  uint32_t *t = nullptr;
  if (MODE == 1) {
    uint32_t o = (uint32_t)scan[w];
    off[w] = o;
    if (w + 1 == n_unique) off[n_unique] = (uint32_t)(scan[w] + lens[w]);
    if (lens[w] == 0) return;
    t = tok + o;
    t[0] = space_id;
  }
  while (q < n && !space_at(s, q, n, &l)) {
    uint32_t cp = decode_unit(s, q, n, &l);
    q += l;
    if (cp == INVALID_CP) continue;
    uint32_t id = cp2id[cp];
    if (id == NO_ID) continue;
    kept++;
    if (MODE == 1) t[kept] = id;
  }
  if (MODE == 0) lens[w] = kept ? kept + 1 : 0;
}

// ------------------------------------------------------------------------------------------
// exclusive scan of uint64 (3 launches; n up to ~2^31)
// ------------------------------------------------------------------------------------------
constexpr int SCAN_T = 256, SCAN_I = 8, SCAN_B = SCAN_T * SCAN_I;

__device__ __forceinline__ unsigned long long block_excl_scan(unsigned long long v, unsigned long long *total) {
  __shared__ unsigned long long wsum[SCAN_T / 32];
  __shared__ unsigned long long wtot;
  unsigned lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  unsigned long long x = v;
  for (int o = 1; o < 32; o <<= 1) {
    unsigned long long y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= (unsigned)o) x += y;
  }
  if (lane == 31) wsum[wid] = x;
  __syncthreads();
  if (wid == 0) {
    unsigned long long s = lane < SCAN_T / 32 ? wsum[lane] : 0, xs = s;
    for (int o = 1; o < 32; o <<= 1) {
      unsigned long long y = __shfl_up_sync(0xffffffffu, xs, o);
      if (lane >= (unsigned)o) xs += y;
    }
    if (lane < SCAN_T / 32) wsum[lane] = xs - s;
    if (lane == 31) wtot = xs;
  }
  __syncthreads();
  unsigned long long r = x - v + wsum[wid];
  *total = wtot;
  __syncthreads();
  return r;
}

__global__ void __launch_bounds__(SCAN_T) scan_block_sums_kernel(const unsigned long long *__restrict__ in, uint64_t n,
                                                                 unsigned long long *__restrict__ bsum) {
  uint64_t base = (uint64_t)blockIdx.x * SCAN_B + (uint64_t)threadIdx.x * SCAN_I;
  unsigned long long v = 0;
  for (int i = 0; i < SCAN_I; i++)
    if (base + i < n) v += in[base + i];
  unsigned long long tot;
  block_excl_scan(v, &tot);
  if (threadIdx.x == 0) bsum[blockIdx.x] = tot;
}
__global__ void __launch_bounds__(SCAN_T) scan_sums_kernel(unsigned long long *bsum, uint64_t nb,
                                                           unsigned long long *total) {
  unsigned long long carry = 0;
  for (uint64_t base = 0; base < nb; base += SCAN_T) {
    uint64_t i = base + threadIdx.x;
    unsigned long long v = i < nb ? bsum[i] : 0, tot;
    unsigned long long e = block_excl_scan(v, &tot);
    if (i < nb) bsum[i] = carry + e;
    carry += tot;
  }
  if (threadIdx.x == 0) *total = carry;
}
__global__ void __launch_bounds__(SCAN_T) scan_final_kernel(const unsigned long long *__restrict__ in, uint64_t n,
                                                            const unsigned long long *__restrict__ bsum,
                                                            unsigned long long *__restrict__ out) {
  uint64_t base = (uint64_t)blockIdx.x * SCAN_B + (uint64_t)threadIdx.x * SCAN_I;
  unsigned long long a[SCAN_I], v = 0;
  for (int i = 0; i < SCAN_I; i++) { a[i] = base + i < n ? in[base + i] : 0; v += a[i]; }
  unsigned long long tot;
  unsigned long long e = block_excl_scan(v, &tot) + bsum[blockIdx.x];
  for (int i = 0; i < SCAN_I; i++) {
    if (base + i < n) out[base + i] = e;
    e += a[i];
  }
}

// ------------------------------------------------------------------------------------------
// phase 3: the pair-count scan (headline kernel): packed tokens -> pair table.
// Algorithmic bytes per launch: 4 T (tokens) + 4 U (offsets) + 8 U (frequencies).
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) pair_hist_kernel(const uint32_t *__restrict__ tok,
                                                        const uint32_t *__restrict__ off,
                                                        const uint64_t *__restrict__ freq, uint64_t n_words,
                                                        PairTab tab) {
  uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  const uint64_t half = tab_slots(tab) / 2;
  const uint32_t key_limit = (uint32_t)(half < 0xffffffffull ? half : 0xffffffffull);
  for (uint64_t w = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; w < n_words; w += stride) {
    // a table that is already half full will be rejected by the host anyway: stop early
    if (__ldcg(tab.overflow) || __ldcg(tab.n_keys) > key_limit) { atomicExch(tab.overflow, 1u); return; }
    uint32_t o = off[w], cap = off[w + 1] - o;
    if (cap < 2) continue;
    long long f = (long long)freq[w];
    for_each_pair(tok + o, cap, [&](uint64_t key, uint64_t mult) { pair_add(tab, key, (long long)mult * f); });
  }
}

// fullest partition of the table (one block per partition)
__global__ void __launch_bounds__(256) part_occ_kernel(PairTab tab, uint32_t *max_occ) {
  __shared__ uint32_t s_n;
  if (threadIdx.x == 0) s_n = 0;
  __syncthreads();
  const uint64_t base = (uint64_t)blockIdx.x * ((uint64_t)tab.rmask + 1);
  uint32_t n = 0;
  for (uint32_t i = threadIdx.x; i <= tab.rmask; i += blockDim.x) n += tab.keys[base + i] != PK_EMPTY ? 1u : 0u;
  for (int o = 16; o > 0; o >>= 1) n += __shfl_xor_sync(0xffffffffu, n, o);
  if ((threadIdx.x & 31) == 0 && n) atomicAdd(&s_n, n);
  __syncthreads();
  if (threadIdx.x == 0) atomicMax(max_occ, s_n);
}

__global__ void pair_dump_kernel(const unsigned long long *__restrict__ keys, const unsigned long long *__restrict__ cnts,
                                 uint64_t cap, unsigned long long *cursor, uint64_t out_cap,
                                 unsigned long long *okeys, unsigned long long *ocnts) {
  uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < cap; i += stride) {
    if (keys[i] == PK_EMPTY || cnts[i] == 0) continue;
    unsigned long long idx = atomicAdd(cursor, 1ull);
    if (idx < out_cap) { okeys[idx] = keys[i]; ocnts[idx] = cnts[i]; }
  }
}

#include "merge_loop.cuh"

// ------------------------------------------------------------------------------------------
// compaction of the packed words: drop tombstones and words with fewer than 2 live tokens
// ------------------------------------------------------------------------------------------
__global__ void compact_len_kernel(const uint32_t *__restrict__ tok, const uint32_t *__restrict__ off,
                                   uint64_t n_words, unsigned long long *__restrict__ packed) {
  uint64_t w = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (w >= n_words) return;
  uint32_t o = off[w];
  uint32_t live = live_len(tok + o, off[w + 1] - o);
  packed[w] = live >= 2 ? ((1ull << 32) | live) : 0ull;  // hi: keeps a word, lo: its tokens
}
__global__ void compact_copy_kernel(const uint32_t *__restrict__ tok, const uint32_t *__restrict__ off,
                                    const uint64_t *__restrict__ freq, uint64_t n_words,
                                    const unsigned long long *__restrict__ packed,
                                    const unsigned long long *__restrict__ scan, uint32_t *__restrict__ ntok,
                                    uint32_t *__restrict__ noff, uint64_t *__restrict__ nfreq) {
  uint64_t w = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (w >= n_words) return;
  unsigned long long p = packed[w];
  if (p == 0) return;
  uint32_t live = (uint32_t)p, nw = (uint32_t)(scan[w] >> 32), no = (uint32_t)scan[w];
  const uint32_t *t = tok + off[w];
  for (uint32_t i = 0; i < live; i++) ntok[no + i] = t[i];
  noff[nw] = no;
  nfreq[nw] = freq[w];
}
__global__ void set_u32_kernel(uint32_t *p, uint32_t v) { *p = v; }

// synthetic packed words for roofline runs of the scan kernel
__global__ void synth_words_kernel(uint32_t *tok, uint32_t *off, uint64_t *freq, uint64_t n_words, uint32_t len,
                                   uint32_t alphabet, uint64_t seed, uint32_t n_first) {
  uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  for (uint64_t w = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; w <= n_words; w += stride) {
    off[w] = (uint32_t)(w * len);
    if (w == n_words) break;
    freq[w] = 1 + (mix64(w ^ seed) & 7);
    uint64_t r = mix64(w * 0x9E3779B97F4A7C15ull + seed);
    tok[w * len] = 4 + (uint32_t)(w % n_first);  // word-initial tokens, never elsewhere (the role of "▁")
    for (uint32_t i = 1; i < len; i++) {
      r = r * 6364136223846793005ull + 1442695040888963407ull;
      tok[w * len + i] = 4 + n_first + (uint32_t)((r >> 33) % alphabet);
    }
  }
}

// ------------------------------------------------------------------------------------------
// host side helpers
// ------------------------------------------------------------------------------------------
int grid_for(yttm_ctx *c, uint64_t n, int threads, int per_sm) {
  uint64_t need = (n + threads - 1) / threads;
  uint64_t cap = (uint64_t)c->n_sm * per_sm;
  return (int)std::max<uint64_t>(1, std::min(need, cap));
}

int device_scan(yttm_ctx *c, const unsigned long long *in, uint64_t n, unsigned long long *out,
                unsigned long long *d_total) {
  uint64_t nb = (n + SCAN_B - 1) / SCAN_B;
  YT_CUDA(c, c->scan_tmp.reserve((nb + 1) * 8));
  auto *bs = c->scan_tmp.as<unsigned long long>();
  scan_block_sums_kernel<<<(unsigned)nb, SCAN_T, 0, c->stream>>>(in, n, bs);
  scan_sums_kernel<<<1, SCAN_T, 0, c->stream>>>(bs, nb, d_total);
  scan_final_kernel<<<(unsigned)nb, SCAN_T, 0, c->stream>>>(in, n, bs, out);
  c->launches += 3;
  YT_CUDA(c, cudaGetLastError());
  return 0;
}

PairTab tab_of(yttm_ctx *c) {
  PairTab t;
  t.keys = c->pkey.as<unsigned long long>();
  t.cnts = c->pcnt.as<unsigned long long>();
  t.rmask = c->p_rmask;
  t.nparts = c->p_nparts;
  YtLoopCtl *ctl = c->ctl.as<YtLoopCtl>();
  t.n_keys = &ctl->n_keys;
  t.overflow = &ctl->overflow;
  return t;
}

// Load factor (percent) above which the merge loop leaves for a rebuild; a rebuilt table is accepted at half of it.
// Default 50 / 25: since round 2 a block sweeps only its own partition, so a roomier table costs little and keeps the
// probe chains of the owners' updates short.  YTTM_PAIR_MAX_LOAD_PCT = 30..90 is an A/B knob.
static uint64_t pair_max_load_pct() {
  return (uint64_t)ytc::env_int("YTTM_PAIR_MAX_LOAD_PCT", 50, 30, 90);
}
// smallest pair table; YTTM_PAIR_CAP_FLOOR lowers it so that tests reach the rebuild / overflow paths on tiny inputs
// (pair_cap_floor_knob: its value, 0 when unset)
static int pair_cap_floor_knob() { return ytc::env_int("YTTM_PAIR_CAP_FLOOR", 0, 16, INT_MAX); }
static uint64_t pair_cap_floor() {
  const int v = pair_cap_floor_knob();
  return v ? ytc::pow2ceil((uint64_t)v) : 1u << 16;
}

// Launch geometry of the cooperative merge loop: one block per SM, all co-resident, with (almost) all of the SM's
// shared memory as the tile buffer.  Fixed per context before the first table is built, because the pair table has one
// partition per block.
// The knobs that shape that geometry and the exchange buffer, read once per context (yttm_geometry_knobs lists them)
constexpr const char *KNOB_STAGES = "YTTM_STAGES", *KNOB_LOOP_THREADS = "YTTM_LOOP_THREADS",
                     *KNOB_XQ_SEG_CAP = "YTTM_XQ_SEG_CAP";
constexpr int LOOP_SMEM_HEAD = (XQ_MAX_WORLD * XQ_MAX_BLOCKS + 4) * 4 + 2 * CLAIM_WORDS * 4 + (int)LOOP_FRONT_BYTES;  // segment prefix + claim bitmaps + front
int ensure_loop_geometry(yttm_ctx *c) {
  if (c->loop_blocks) return 0;
  int optin = 0;
  YT_CUDA(c, cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, c->device));
  int dyn = optin - 4096;  // static shared memory of the kernel (~1.5 KB) + margin
  if (dyn < 64 * 1024) YT_FAIL(c, "merge_loop_kernel: not enough shared memory per block");
  c->loop_smem = dyn;
  const int tile_bytes = dyn - LOOP_SMEM_HEAD;
  // RESIDENT tile: per word 4 B offset + 8 B frequency (kept in shared memory too, so a rewritten
  // word costs no L2 round trip for its frequency), the rest token slots
  c->loop_word_cap = std::min<uint32_t>((uint32_t)(tile_bytes / 24 - 2), CLAIM_WORDS * 32 - 1) & ~1u;
  c->loop_tok_cap = (uint32_t)((tile_bytes - 12 * (c->loop_word_cap + 2)) / 4) & ~3u;
  // STREAMING: n_stage stages; a stage holds a window of q slots plus the overhang of its last
  // word (words of up to q/4 slots stay on the shared-memory path) and at most q/2 + 1 offsets
  {
    // H100: 2, 3 and 4 stages scan within 1.5 % of each other (tools/probe_scan.py, YTTM_STAGES)
    const int n_stage = ytc::env_int(KNOB_STAGES, 2, 2, MAX_STAGES);
    const uint32_t per_stage = (uint32_t)(tile_bytes / n_stage / 4) & ~3u;  // uint32 per stage
    // tokens: q + q/4 + 8, offsets: q/2 + 16  ->  q * 1.75 + 24 <= per_stage
    uint32_t q = (uint32_t)((per_stage - 24) / 1.75);
    q &= ~15u;
    c->loop_stages = n_stage;
    c->loop_stream_q = q;
    c->loop_stream_word_cap = (q / 2 + 16) & ~3u;
    c->loop_stream_tok_cap = (per_stage - c->loop_stream_word_cap) & ~3u;
  }
  YT_CUDA(c, cudaFuncSetAttribute(merge_loop_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, dyn));
  // H100, 100 MB Zipf: 8.1 us per merge with 512 threads (128 registers), 11.3 with 1024 (64, spills)
  // tests: smaller blocks change how the scans and the drain split their work (512 at most: the kernel's launch bounds)
  const int threads = ytc::env_int(KNOB_LOOP_THREADS, 512, 64, 512) / 32 * 32;
  int per_sm = 0;
  YT_CUDA(c, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, merge_loop_kernel, threads, dyn));
  if (per_sm < 1) YT_FAIL(c, "merge_loop_kernel does not fit on an SM");
  c->loop_threads = threads;
  // (a refresh of the front takes FRONT_TOP pairs from every block's partition and must leave room for new pairs)
  const int blocks = std::min(std::min(c->n_sm, XQ_MAX_BLOCKS), (int)(FRONT_FILL / FRONT_TOP));
  if (c->xq_nblocks && (int)c->xq_nblocks != blocks) YT_FAIL(c, "merge loop geometry differs from the exchange buffer's");
  c->loop_blocks = blocks;
  return 0;
}

// Exchange buffer of the merge loop.  Entries per (sender, block) segment: YTTM_XQ_SEG_CAP (tests use tiny values
// to reach the overflow -> rebuild path); a merge whose count changes do not fit is still applied to the words and
// the table is rebuilt from them, so the capacity is a performance knob, not a limit.  It sizes a buffer whose address
// the other ranks of a job hold from yttm_train_dist_connect on, so it is read once per context, like the geometry.
int xq_alloc(yttm_ctx *c, uint32_t me, uint32_t world) {
  if (ensure_loop_geometry(c)) return 1;
  const uint32_t seg_cap = (uint32_t)ytc::env_int(KNOB_XQ_SEG_CAP, 8192, 4, INT_MAX);
  c->xq_world = world; c->xq_me = me; c->xq_seg_cap = seg_cap; c->xq_nblocks = (uint32_t)c->loop_blocks;
  c->xq_per_sender = (sizeof(XqHdr) + (uint64_t)c->xq_nblocks * seg_cap * sizeof(uint4) + 255) / 256 * 256;
  c->xq_bytes = 2ull * world * c->xq_per_sender;
  YT_CUDA(c, c->xq_buf.reserve(c->xq_bytes));
  YT_CUDA(c, c->xq_arrive.reserve(64));
  // entries start as all-ones (a stamp no round uses), count words as round 0
  YT_CUDA(c, cudaMemsetAsync(c->xq_buf.p, 0xff, c->xq_bytes, c->stream));
  for (uint32_t k = 0; k < 2 * world; k++)
    YT_CUDA(c, cudaMemsetAsync(c->xq_buf.as<unsigned char>() + k * c->xq_per_sender, 0, offsetof(XqHdr, places), c->stream));   // count words: round 0; entry places stay all-ones
  YT_CUDA(c, cudaMemsetAsync(c->xq_arrive.p, 0, 64, c->stream));
  YT_CUDA(c, cudaStreamSynchronize(c->stream));
  for (int d = 0; d < XQ_MAX_WORLD; d++) c->xq_peer[d] = nullptr;
  c->xq_peer[me] = c->xq_buf.p;
  c->xq_connected = world == 1;
  return 0;
}
static unsigned long long xq_spin_limit_ns() {
  return (unsigned long long)ytc::env_int("YTTM_XQ_TIMEOUT_MS", 30000, 1, INT_MAX) * 1000000ull;
}
int xq_args(yttm_ctx *c, LoopArgs *a) {
  if (!c->xq_buf.p && xq_alloc(c, 0, 1)) return 1;
  if (!c->xq_connected) YT_FAIL(c, "distributed training: yttm_train_dist_connect has not run");
  for (int d = 0; d < XQ_MAX_WORLD; d++) a->xq.base[d] = static_cast<unsigned char *>(c->xq_peer[d < (int)c->xq_world ? d : (int)c->xq_me]);
  a->xq.world = c->xq_world; a->xq.me = c->xq_me; a->xq.nblocks = c->xq_nblocks; a->xq.seg_cap = c->xq_seg_cap;
  a->xq.per_sender = c->xq_per_sender;
  a->spin_limit_ns = xq_spin_limit_ns();
  return 0;
}

// capacity -> (partitions, slots per partition): one partition per loop block, R a power of two >= 16
static void set_table_shape(yttm_ctx *c, uint64_t want_slots) {
  const uint64_t parts = (uint64_t)c->loop_blocks;
  const uint64_t R = std::max<uint64_t>(ytc::pow2ceil((want_slots + parts - 1) / parts), 16);
  c->p_nparts = (uint32_t)parts;
  c->p_rmask = (uint32_t)(R - 1);
  c->pcap = parts * R;
}

// One attempt: clear a table of >= want_slots slots and histogram the local packed words into it; then, in a
// multi-GPU job, one exchange round adds every other rank's pairs (all ranks run this in lockstep with the same
// want_slots).  *ok: the table is usable (nothing dropped, load factor and fullest partition within bounds) — a
// function of the key set and the shape only, hence the same verdict on every rank.
static int build_table_once(yttm_ctx *c, uint64_t want_slots, bool *ok) {
  set_table_shape(c, want_slots);
  const uint64_t cap = c->pcap;
  YT_CUDA(c, c->pkey.reserve(cap * 8));
  YT_CUDA(c, c->pcnt.reserve(cap * 8));
  YT_CUDA(c, cudaMemsetAsync(c->pkey.p, 0xff, cap * 8, c->stream));
  YT_CUDA(c, cudaMemsetAsync(c->pcnt.p, 0, cap * 8, c->stream));
  YtLoopCtl *ctl = c->ctl.as<YtLoopCtl>();
  YT_CUDA(c, cudaMemsetAsync(&ctl->n_keys, 0, 8, c->stream));  // n_keys + overflow
  YT_CUDA(c, cudaMemsetAsync(&ctl->xq_flags, 0, 8, c->stream));  // xq_flags + max_part_occ
  if (c->n_words) {
    pair_hist_kernel<<<grid_for(c, c->n_words, 256, 8), 256, 0, c->stream>>>(
        c->tok[c->cur].as<uint32_t>(), c->off[c->cur].as<uint32_t>(), c->freq[c->cur].as<uint64_t>(), c->n_words,
        tab_of(c));
    c->launches++;
  }
  uint32_t peer_flags = 0;
  if (c->xq_world > 1) {
    LoopArgs a{};
    if (xq_args(c, &a)) return 1;
    a.tab = tab_of(c);
    a.ctl = ctl;
    uint32_t round = 0;
    YT_CUDA(c, cudaMemcpyAsync(&round, &ctl->xq_round, 4, cudaMemcpyDeviceToHost, c->stream));
    // the rounds publish a SNAPSHOT of the local histogram: absorbing the peers' pairs changes the table itself
    YT_CUDA(c, c->scratch_key.reserve(cap * 8));
    YT_CUDA(c, c->scratch_cnt.reserve(cap * 8));
    YT_CUDA(c, cudaMemcpyAsync(c->scratch_key.p, c->pkey.p, cap * 8, cudaMemcpyDeviceToDevice, c->stream));
    YT_CUDA(c, cudaMemcpyAsync(c->scratch_cnt.p, c->pcnt.p, cap * 8, cudaMemcpyDeviceToDevice, c->stream));
    YT_CUDA(c, cudaStreamSynchronize(c->stream));
    LoopArgs snap = a;
    snap.tab.keys = c->scratch_key.as<unsigned long long>();
    snap.tab.cnts = c->scratch_cnt.as<unsigned long long>();
    for (uint32_t chunk = 0;; chunk++) {  // every rank runs the same number of rounds: "more" is OR-ed over all senders
      round += 1;
      xq_publish_table_kernel<<<c->p_nparts, 256, 0, c->stream>>>(snap, round, chunk, &ctl->overflow);
      xq_absorb_kernel<<<c->p_nparts, 256, (XQ_MAX_WORLD * XQ_MAX_BLOCKS + 4) * 4, c->stream>>>(a, round);
      c->launches += 2;
      uint32_t f = 0;
      YT_CUDA(c, cudaMemcpyAsync(&f, &ctl->xq_flags, 4, cudaMemcpyDeviceToHost, c->stream));
      YT_CUDA(c, cudaStreamSynchronize(c->stream));
      peer_flags |= f;
      if (!(f & XQF_MORE)) break;
      if (chunk > 100000) YT_FAIL(c, "distributed table build: too many exchange rounds");
      YT_CUDA(c, cudaMemsetAsync(&ctl->xq_flags, 0, 4, c->stream));
    }
  }
  part_occ_kernel<<<c->p_nparts, 256, 0, c->stream>>>(tab_of(c), &ctl->max_part_occ);
  c->launches++;
  YT_CUDA(c, cudaGetLastError());
  uint32_t h[2], g[2];
  YT_CUDA(c, cudaMemcpyAsync(h, &ctl->n_keys, 8, cudaMemcpyDeviceToHost, c->stream));
  YT_CUDA(c, cudaMemcpyAsync(g, &ctl->xq_flags, 8, cudaMemcpyDeviceToHost, c->stream));
  YT_CUDA(c, cudaStreamSynchronize(c->stream));
  peer_flags |= g[0];
  const uint64_t R = (uint64_t)c->p_rmask + 1;
  // local overflow is rank-specific, but it reaches every rank as XQF_OVERFLOW of this rank's round
  // accept at half the load the loop leaves at, globally and in the fullest partition (+ 1/8 slack for imbalance)
  *ok = !h[1] && !(peer_flags & XQF_OVERFLOW) && (uint64_t)h[0] * 200 <= cap * pair_max_load_pct() &&
        (uint64_t)g[1] * 200 <= R * (pair_max_load_pct() + 25);
  if (*ok) { c->stats.n_pairs = h[0]; c->stats.table_capacity = cap; }
  return 0;
}

// (Re)build the pair table from the current packed words: grows it until build_table_once accepts.
int ensure_ctl(yttm_ctx *c) {
  if (c->ctl.p) return 0;
  YT_CUDA(c, c->ctl.reserve(sizeof(YtLoopCtl)));
  YT_CUDA(c, cudaMemsetAsync(c->ctl.p, 0, sizeof(YtLoopCtl), c->stream));
  return 0;
}
int rebuild_pair_table(yttm_ctx *c, uint64_t min_cap) {
  if (ensure_loop_geometry(c)) return 1;
  if (ensure_ctl(c)) return 1;
  uint64_t cap = std::max<uint64_t>(ytc::pow2ceil(min_cap), pair_cap_floor());
  for (int attempt = 0; attempt < 28; attempt++) {
    bool ok = false;
    if (build_table_once(c, cap, &ok)) return 1;
    if (ok) return 0;
    cap *= 2;
  }
  YT_FAIL(c, "pair table: could not reach the target load factor");
}

// Compact the packed words into the other buffer set.
int compact_words(yttm_ctx *c) {
  if (c->n_words == 0) return 0;
  uint64_t nw = c->n_words;
  int src = c->cur, dst = 1 - c->cur;
  YT_CUDA(c, c->wlen.reserve((nw + 1) * 8));
  YT_CUDA(c, c->wpos.reserve((nw + 1) * 8));
  auto *packed = c->wlen.as<unsigned long long>();
  auto *scan = c->wpos.as<unsigned long long>();
  YT_CUDA(c, c->counters.reserve(64));
  auto *d_total = c->counters.as<unsigned long long>() + 4;
  unsigned nb = (unsigned)((nw + 255) / 256);
  compact_len_kernel<<<nb, 256, 0, c->stream>>>(c->tok[src].as<uint32_t>(), c->off[src].as<uint32_t>(), nw, packed);
  c->launches++;
  if (device_scan(c, packed, nw, scan, d_total)) return 1;
  unsigned long long tot;
  YT_CUDA(c, cudaMemcpyAsync(&tot, d_total, 8, cudaMemcpyDeviceToHost, c->stream));
  YT_CUDA(c, cudaStreamSynchronize(c->stream));
  uint64_t new_words = tot >> 32, new_slots = tot & 0xffffffffull;
  YT_CUDA(c, c->tok[dst].reserve((new_slots + 4) * 4));
  YT_CUDA(c, c->off[dst].reserve((new_words + 2) * 4));
  YT_CUDA(c, c->freq[dst].reserve((new_words + 1) * 8));
  compact_copy_kernel<<<nb, 256, 0, c->stream>>>(c->tok[src].as<uint32_t>(), c->off[src].as<uint32_t>(),
                                                  c->freq[src].as<uint64_t>(), nw, packed, scan,
                                                  c->tok[dst].as<uint32_t>(), c->off[dst].as<uint32_t>(),
                                                  c->freq[dst].as<uint64_t>());
  set_u32_kernel<<<1, 1, 0, c->stream>>>(c->off[dst].as<uint32_t>() + new_words, (uint32_t)new_slots);
  c->launches += 2;
  YT_CUDA(c, cudaGetLastError());
  c->cur = dst;
  c->n_words = new_words;
  c->n_slots = new_slots;
  return 0;
}

// Decide how the merge loop sees the packed words: RESIDENT (one tile per block, kept in shared
// memory for the whole launch) when every tile fits, else STREAMING tiles of `q` token slots.
int plan_tiles(yttm_ctx *c, LoopArgs *a) {
  const uint32_t *off = c->off[c->cur].as<uint32_t>();
  a->smem_tok_cap = c->loop_tok_cap;
  a->smem_word_cap = c->loop_word_cap;
  a->resident = 0;
  a->n_tiles = 0;
  a->tile_desc = nullptr;
  a->stream_tok_cap = c->loop_stream_tok_cap;
  a->stream_word_cap = c->loop_stream_word_cap;
  a->defer = nullptr;
  a->defer_cap = 0;
  a->n_stage = (uint32_t)c->loop_stages;
  c->loop_resident = 0;
  if (c->n_words == 0 || c->n_slots == 0) return 0;
  YT_CUDA(c, c->counters.reserve(64));
  uint32_t *d_stats = reinterpret_cast<uint32_t *>(c->counters.as<unsigned long long>() + 7);
  const bool force_stream = ytc::env_set("YTTM_FORCE_STREAM");
  const uint32_t stream_q = (uint32_t)ytc::env_int("YTTM_STREAM_Q", (int)c->loop_stream_q, 1, INT_MAX);
  for (int pass = force_stream ? 1 : 0; pass < 2; pass++) {
    uint64_t q = pass == 0 ? (c->n_slots + c->loop_blocks - 1) / c->loop_blocks : stream_q;
    if (q == 0) q = 1;
    uint64_t n_tiles = (c->n_slots + q - 1) / q;
    YT_CUDA(c, c->tiles.reserve((n_tiles + 2) * 8));
    unsigned nb = (unsigned)((c->n_words + 255) / 256);
    tile_desc_kernel<<<nb, 256, 0, c->stream>>>(off, c->n_words, (uint32_t)q, (uint32_t)n_tiles,
                                                 c->tiles.as<uint2>());
    c->launches++;
    a->tile_desc = c->tiles.as<uint2>();
    a->n_tiles = (uint32_t)n_tiles;
    if (pass == 1) {
      // words per block and merge on the deferred path; beyond it the direct pass takes over
      a->defer_cap = (uint32_t)ytc::env_int("YTTM_DEFER_CAP", 8192, 1, INT_MAX);
      YT_CUDA(c, c->defer.reserve((size_t)c->loop_blocks * a->defer_cap * sizeof(uint4)));
      a->defer = c->defer.as<uint4>();
      break;
    }
    YT_CUDA(c, cudaMemsetAsync(d_stats, 0, 8, c->stream));
    tile_stats_kernel<<<(unsigned)((n_tiles + 255) / 256), 256, 0, c->stream>>>(c->tiles.as<uint2>(),
                                                                                  (uint32_t)n_tiles, d_stats);
    c->launches++;
    uint32_t h[2];
    YT_CUDA(c, cudaMemcpyAsync(h, d_stats, 8, cudaMemcpyDeviceToHost, c->stream));
    YT_CUDA(c, cudaStreamSynchronize(c->stream));
    // RESIDENT if the largest tile fits the block's tile bytes: 4 B per token slot (rounded up to 16 B) + 12 B per word
    // (+ 2 sentinel offsets); the split between tokens and words follows the corpus
    {
      const uint64_t tok = ((uint64_t)h[0] + 7) & ~3ull, wrd = ((uint64_t)h[1] + 3) & ~1ull;
      const uint64_t tile_bytes = (uint64_t)c->loop_smem - LOOP_SMEM_HEAD;
      if (wrd <= CLAIM_WORDS * 32 - 1 && tok * 4 + (wrd + 2) * 12 + 64 <= tile_bytes) {
        a->smem_tok_cap = (uint32_t)tok;
        a->smem_word_cap = (uint32_t)wrd;
        a->resident = 1; c->loop_resident = 1;
        break;
      }
    }
  }
  YT_CUDA(c, cudaGetLastError());
  return 0;
}

// every device buffer the context owns
std::vector<ytc::DevBuf *> ctx_bufs(yttm_ctx *c) {
  return {&c->text_buf, &c->hist, &c->cp2id, &c->wkey, &c->wcnt, &c->wpos, &c->wfreq, &c->wlen, &c->scan_tmp,
          &c->counters, &c->tok[0], &c->tok[1], &c->off[0], &c->off[1], &c->freq[0], &c->freq[1], &c->pkey, &c->pcnt,
          &c->scratch_key, &c->scratch_cnt, &c->ctl, &c->frontbuf, &c->tiles, &c->defer, &c->d_rules, &c->d_rfreq,
          &c->xq_arrive, &c->xq_buf, &c->feed_dev[0], &c->feed_dev[1], &c->fkey, &c->fcnt, &c->arena};
}

// The device memory high-water mark of the current training ("dev_peak_bytes"): sampled after every phase and every fed
// piece, it shows whether a corpus sat on the device.
void note_peak(yttm_ctx *c) {
  uint64_t sum = 0;
  for (auto *b : ctx_bufs(c)) sum += b->cap;
  c->dev_peak = std::max(c->dev_peak, sum);
}

}  // namespace

const char *const yttm_geometry_knobs[] = {KNOB_STAGES, KNOB_LOOP_THREADS, KNOB_XQ_SEG_CAP, "YT_EMU_SMS", nullptr};

thread_local std::string g_yttm_create_error;

int yttm_device_scan_u64(yttm_ctx *c, const unsigned long long *in, uint64_t n, unsigned long long *out,
                         unsigned long long *d_total) {
  return device_scan(c, in, n, out, d_total);
}

// Whether train_bpe / learn_bpe_from_string feed a corpus of n bytes (UINT64_MAX: size unknown) rather than load it.
// The in-memory path holds the corpus, a word table of up to two slots of 16 B per 16 corpus bytes (1 GB at most) and
// the tokens of the unique words at once, so a corpus above a third of the device's free memory at the start of the
// training is fed (DESIGN §3).  YTTM_TRAIN_FEED_ABOVE (bytes) replaces that threshold.
bool yttm_train_feed_selected(yttm_ctx *c, uint64_t n) {
  if (n == UINT64_MAX) return true;
  if (const char *e = std::getenv("YTTM_TRAIN_FEED_ABOVE")) return n > std::strtoull(e, nullptr, 10);
#ifndef YT_SIMT_EMU
  size_t free_b = 0, total_b = 0;
  if (cudaSetDevice(c->device) != cudaSuccess || cudaMemGetInfo(&free_b, &total_b) != cudaSuccess) return false;
  return n > free_b / 3;
#else
  return false;   // tests/emul/simt: no device memory to ask about; the knob selects
#endif
}

// =============================================================================================
// C ABI
// =============================================================================================
extern "C" {

int yttm_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) return 0;
  return n;
}

int yttm_ctx_create(int device, yttm_ctx **out) {
  *out = nullptr;
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess || n == 0) {
    g_yttm_create_error = std::string("yttm_b200: no CUDA device available (") +
                          (e == cudaSuccess ? "device count is 0" : cudaGetErrorString(e)) +
                          "); this library has no CPU fallback";
    return 1;
  }
  if (device < 0 || device >= n) { g_yttm_create_error = "yttm_b200: bad device index"; return 1; }
  if ((e = cudaSetDevice(device)) != cudaSuccess) { g_yttm_create_error = cudaGetErrorString(e); return 1; }
  yttm_ctx *c = new yttm_ctx();
  c->device = device;
  cudaDeviceGetAttribute(&c->n_sm, cudaDevAttrMultiProcessorCount, device);
  if ((e = cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking)) != cudaSuccess) {
    g_yttm_create_error = cudaGetErrorString(e);
    delete c;
    return 1;
  }
  *out = c;
  return 0;
}

void yttm_ctx_destroy(yttm_ctx *c) {
  if (!c) return;
  cudaSetDevice(c->device);
  cudaStreamSynchronize(c->stream);
  if (c->stream2) cudaStreamSynchronize(c->stream2);
  for (int d = 0; d < 8; d++)
    if (c->xq_peer_ipc[d] && c->xq_peer[d]) { cudaIpcCloseMemHandle(c->xq_peer[d]); c->xq_peer[d] = nullptr; }
  for (auto *b : ctx_bufs(c)) b->release();
  for (auto &kv : c->timers) { if (kv.second.a) cudaEventDestroy(kv.second.a); if (kv.second.b) cudaEventDestroy(kv.second.b); }
  for (int s = 0; s < 2; s++) {
    if (c->feed_stage[s]) cudaFreeHost(c->feed_stage[s]);
    if (c->ev_feed_copied[s]) cudaEventDestroy(c->ev_feed_copied[s]);
    if (c->ev_feed_done[s]) cudaEventDestroy(c->ev_feed_done[s]);
  }
  if (c->stream2) cudaStreamDestroy(c->stream2);
  if (c->ev_pipe) cudaEventDestroy(c->ev_pipe);
  cudaStreamDestroy(c->stream);
  delete c;
}

const char *yttm_last_error(const yttm_ctx *c) { return c ? c->err.c_str() : g_yttm_create_error.c_str(); }

double yttm_stage_ms(const yttm_ctx *c, const char *stage) {
  // block 0's share of a merge (merge_loop.cuh): drain = wait for the count words + entries + new pairs; elect = front
  // scan (+ refreshes); apply = token scan + rewrites + count word; partition = parked entries into the table
  static const char *ph[] = {"loop_drain", "loop_elect", "loop_apply", "loop_partition"};
  for (int i = 0; i < 4; i++)
    if (!std::strcmp(stage, ph[i])) return c->loop_phase_ms[i];
  if (!std::strcmp(stage, "loop_iters")) return (double)c->loop_iters;
  if (!std::strcmp(stage, "xq_round")) return (double)c->loop_xq_round;   // exchange rounds of the context so far
  if (!std::strcmp(stage, "enc_chunks")) return c->enc_chunks;
  if (!std::strcmp(stage, "loop_refreshes")) return (double)c->loop_sweeps;
  if (!std::strcmp(stage, "loop_launches")) return (double)c->loop_relaunches;
  if (!std::strcmp(stage, "table_capacity")) return (double)c->pcap;
  if (!std::strcmp(stage, "loop_resident")) return (double)c->loop_resident;
  if (!std::strcmp(stage, "feed_pieces")) return (double)c->feed_pieces;
  if (!std::strcmp(stage, "dev_peak_bytes")) return (double)c->dev_peak;
  return ytc::timer_ms(const_cast<yttm_ctx *>(c), stage);
}
uint64_t yttm_launch_count(const yttm_ctx *c) { return c->launches; }

// Length of the longest prefix of [p, p + n) that ends with a whitespace byte (space, \t .. \r), 0 if there is none.
// A piece of the corpus cut there is self-contained for both byte passes: no UTF-8 sequence and no word crosses its
// end (a whitespace byte is a whole unit), and what precedes its start is a space (the kernels' view of "outside the
// text").
static uint64_t piece_cut(const char *p, uint64_t n) {
  for (uint64_t i = n; i > 0; i--)
    if (is_space_byte((uint8_t)p[i - 1])) return i;
  return 0;
}

static int ensure_stream2(yttm_ctx *c) {
  if (!c->stream2) {
    YT_CUDA(c, cudaStreamCreateWithFlags(&c->stream2, cudaStreamNonBlocking));
    YT_CUDA(c, cudaEventCreateWithFlags(&c->ev_pipe, cudaEventDisableTiming));
  }
  return 0;
}

// The corpus comes from pageable host memory at ~11 GB/s, and the two byte passes over it (code point histogram, word
// split + dedup) need neither each other nor the alphabet: the text is copied in pieces (piece_cut), and both passes
// run on a piece (second stream) while the next one is copied.  Corpora without a whitespace byte in 32 MB fall back
// to one piece.
static int pipelined_load(yttm_ctx *c, uint8_t *dst, const char *src, uint64_t n) {
  if (ensure_stream2(c)) return 1;
  const uint64_t piece = (uint64_t)ytc::env_int("YTTM_TRAIN_PIPELINE_PIECE_KB", 32 << 10, 1, INT_MAX) << 10;   // tests: small pieces
  YT_CUDA(c, c->hist.reserve((CP_LIMIT + 1) * 8));
  YT_CUDA(c, cudaMemsetAsync(c->hist.p, 0, (CP_LIMIT + 1) * 8, c->stream));
  YT_CUDA(c, c->counters.reserve(64));
  auto *counters = c->counters.as<unsigned long long>();
  const uint64_t cap = std::min<uint64_t>(std::max<uint64_t>(ytc::pow2ceil(n / 16 + 1), 1u << 16), 1ull << 26);   // as build_word_table
  YT_CUDA(c, c->wkey.reserve(cap * 8));
  YT_CUDA(c, c->wcnt.reserve(cap * 8));
  YT_CUDA(c, cudaMemsetAsync(c->wkey.p, 0, cap * 8, c->stream));
  YT_CUDA(c, cudaMemsetAsync(c->wcnt.p, 0, cap * 8, c->stream));
  YT_CUDA(c, cudaMemsetAsync(counters, 0, 64, c->stream));
  WordTab wt{c->wkey.as<unsigned long long>(), c->wcnt.as<unsigned long long>(), cap - 1};
  for (uint64_t lo = 0; lo < n;) {
    uint64_t hi = std::min<uint64_t>(n, lo + piece);
    if (hi < n) {
      const uint64_t cut = piece_cut(src + lo, hi - lo);
      hi = cut ? lo + cut : n;
    }
    YT_CUDA(c, cudaMemcpyAsync(dst + lo, src + lo, hi - lo, cudaMemcpyHostToDevice, c->stream));
    YT_CUDA(c, cudaEventRecord(c->ev_pipe, c->stream));
    YT_CUDA(c, cudaStreamWaitEvent(c->stream2, c->ev_pipe, 0));
    char_hist_kernel<<<grid_for(c, (hi - lo) / 16 + 1, 512, 4), 512, 0, c->stream2>>>(dst + lo, hi - lo, c->hist.as<unsigned long long>());
    word_insert_kernel<<<grid_for(c, hi - lo, 256, 8), 256, 0, c->stream2>>>(dst, n, lo, hi, wt, counters, cap / 2);
    c->launches += 2;
    lo = hi;
  }
  YT_CUDA(c, cudaGetLastError());
  c->pipe_hist = true;
  c->pipe_wtab_cap = cap;
  return 0;
}

static int feed_release(yttm_ctx *c);
static int hist_summarise(yttm_ctx *c, uint64_t *data_len, uint64_t *n_distinct);

int yttm_train_load_corpus(yttm_ctx *c, const char *bytes, uint64_t n, int on_device) {
  YT_CUDA(c, cudaSetDevice(c->device));
  if (n >= POS_MASK) YT_FAIL(c, "corpus shard too large (>= 2^40 bytes)");
  // a new training starts: nothing built from an earlier corpus (words, pair table, a pipelined histogram or word
  // table that no char_hist / build consumed) and no stage time of an earlier training may pass for this one's
  c->n_text = n;
  c->have_alphabet = false;
  c->pipe_hist = false;
  c->pipe_wtab_cap = 0;
  c->n_words = c->n_slots = c->n_unique = c->n_word_occ = 0;
  c->pcap = 0;
  c->stats = yttm_train_stats{};
  ytc::timers_reset(c);
  if ((c->feeding || c->arena.p) && feed_release(c)) return 1;   // an abandoned feed
  c->fed_words = false;
  c->feed_pieces = 0;
  c->dev_peak = 0;
  if (on_device) {
    c->d_text = reinterpret_cast<const uint8_t *>(bytes);
    c->text_external = true;
    note_peak(c);
    return 0;
  }
  ytc::timer_begin(c, "h2d");
  YT_CUDA(c, c->text_buf.reserve(n + 64));
  uint8_t *base = c->text_buf.as<uint8_t>();
  YT_CUDA(c, cudaMemsetAsync(base, ' ', 16, c->stream));
  YT_CUDA(c, cudaMemsetAsync(base + 16 + n, ' ', 32, c->stream));
  c->d_text = base + 16;
  c->text_external = false;
  // bytes; below 64 MB the passes are too short to be worth a second stream; YTTM_TRAIN_PIPELINE=0: off
  const int pipe_knob = ytc::env_int("YTTM_TRAIN_PIPELINE", 64 << 20, 0, INT_MAX);
  const uint64_t pipe_min = pipe_knob > 0 ? (uint64_t)pipe_knob : ~0ull;
  if (n >= pipe_min) { if (pipelined_load(c, base + 16, bytes, n)) return 1; }
  else if (n) YT_CUDA(c, cudaMemcpyAsync(base + 16, bytes, n, cudaMemcpyHostToDevice, c->stream));
  ytc::timer_end(c, "h2d");
  if (c->pipe_hist) {   // the kernels of the last pieces: everything after this call sees them done
    YT_CUDA(c, cudaEventRecord(c->ev_pipe, c->stream2));
    YT_CUDA(c, cudaStreamWaitEvent(c->stream, c->ev_pipe, 0));
  }
  note_peak(c);
  return 0;
}

// ---- fed corpus (include/yttm_b200.h: yttm_train_feed_begin / feed / feed_end) ------------------------------------
// Host side of a piece: bytes gather in staging buffer feed_cur until it holds a nominal piece; the piece then ends
// behind its last whitespace byte (piece_cut) and what follows moves to the other staging buffer.  A piece is copied
// on stream2 and processed (feed_process) when the next piece has been cut, so its copy overlaps the passes of the
// piece before it.

// drops what a feed holds on the device (the feed_end that consumed it or a new training after an abandoned feed)
static int feed_release(yttm_ctx *c) {
  if (c->stream2) YT_CUDA(c, cudaStreamSynchronize(c->stream2));
  YT_CUDA(c, cudaStreamSynchronize(c->stream));
  for (ytc::DevBuf *b : {&c->feed_dev[0], &c->feed_dev[1], &c->fkey, &c->fcnt, &c->arena}) b->release();
  c->feeding = false;
  c->fed_words = false;
  c->feed_pending = -1;
  return 0;
}

// staging buffer s holds at least `need` bytes (its first feed_len bytes kept when it is the one being filled)
static int stage_reserve(yttm_ctx *c, int s, uint64_t need) {
  if (need <= c->feed_stage_cap[s]) return 0;
  const uint64_t cap = std::max<uint64_t>({need, 2 * c->feed_stage_cap[s], c->feed_piece});
  void *p = nullptr;
  YT_CUDA(c, cudaHostAlloc(&p, cap, cudaHostAllocDefault));
  if (s == c->feed_cur && c->feed_len) std::memcpy(p, c->feed_stage[s], c->feed_len);
  if (c->feed_stage[s]) YT_CUDA(c, cudaFreeHost(c->feed_stage[s]));
  c->feed_stage[s] = static_cast<uint8_t *>(p);
  c->feed_stage_cap[s] = cap;
  return 0;
}

// the arena holds its 16 pad bytes + `need` text bytes + 32 pad bytes; its bytes so far move to a larger buffer
static int arena_reserve(yttm_ctx *c, uint64_t need) {
  if (16 + need + 32 <= c->arena.cap) return 0;
  ytc::DevBuf bigger;
  YT_CUDA(c, bigger.reserve(std::max<uint64_t>(16 + need + 32, 2 * c->arena.cap)));
  YT_CUDA(c, cudaMemcpyAsync(bigger.p, c->arena.p, 16 + c->arena_len, cudaMemcpyDeviceToDevice, c->stream));
  YT_CUDA(c, cudaStreamSynchronize(c->stream));
  c->arena.release();
  c->arena = bigger;
  return 0;
}

// the persistent table keeps its load at most 1/2 with `more` further words; a larger table is rehashed from the arena
static int ftab_reserve(yttm_ctx *c, uint64_t more) {
  uint64_t cap = c->feed_fcap;
  while ((c->feed_fn + more) * 2 > cap) cap *= 4;
  if (cap == c->feed_fcap) return 0;
  ytc::DevBuf nk, nc;
  YT_CUDA(c, nk.reserve(cap * 8));
  YT_CUDA(c, nc.reserve(cap * 8));
  YT_CUDA(c, cudaMemsetAsync(nk.p, 0, cap * 8, c->stream));
  YT_CUDA(c, cudaMemsetAsync(nc.p, 0, cap * 8, c->stream));
  WordTab old{c->fkey.as<unsigned long long>(), c->fcnt.as<unsigned long long>(), c->feed_fcap - 1};
  WordTab nt{nk.as<unsigned long long>(), nc.as<unsigned long long>(), cap - 1};
  word_table_rehash_kernel<<<grid_for(c, c->feed_fcap, 256, 8), 256, 0, c->stream>>>(old, nt, c->arena.as<uint8_t>() + 16,
                                                                                   c->arena_len);
  c->launches++;
  YT_CUDA(c, cudaGetLastError());
  YT_CUDA(c, cudaStreamSynchronize(c->stream));
  c->fkey.release(); c->fcnt.release();
  c->fkey = nk; c->fcnt = nc;
  c->feed_fcap = cap;
  return 0;
}

// Phase 1 and the word split of piece buffer s (m bytes), then its distinct words into the persistent table.
static int feed_process(yttm_ctx *c, int s, uint64_t m) {
  const uint8_t *d = c->feed_dev[s].as<uint8_t>();
  auto *counters = c->counters.as<unsigned long long>();
  YT_CUDA(c, cudaStreamWaitEvent(c->stream, c->ev_feed_copied[s], 0));
  char_hist_kernel<<<grid_for(c, m / 16 + 1, 512, 4), 512, 0, c->stream>>>(d, m, c->hist.as<unsigned long long>());
  c->launches++;
  unsigned long long h[6] = {0, 0, 0, 0, 0, 0};
  for (int attempt = 0;; attempt++) {   // a piece that overflows the per-piece table is split again in a larger one
    if (attempt > 10) YT_FAIL(c, "word table: too many retries");
    const uint64_t cap = c->feed_wcap;
    YT_CUDA(c, c->wkey.reserve(cap * 8));
    YT_CUDA(c, c->wcnt.reserve(cap * 8));
    YT_CUDA(c, cudaMemsetAsync(c->wkey.p, 0, cap * 8, c->stream));
    YT_CUDA(c, cudaMemsetAsync(c->wcnt.p, 0, cap * 8, c->stream));
    YT_CUDA(c, cudaMemsetAsync(counters, 0, 64, c->stream));
    WordTab wt{c->wkey.as<unsigned long long>(), c->wcnt.as<unsigned long long>(), cap - 1};
    word_insert_kernel<<<grid_for(c, m, 256, 8), 256, 0, c->stream>>>(d, m, 0, m, wt, counters, cap / 2);
    c->launches++;
    YT_CUDA(c, cudaGetLastError());
    YT_CUDA(c, cudaMemcpyAsync(h, counters, 32, cudaMemcpyDeviceToHost, c->stream));
    YT_CUDA(c, cudaStreamSynchronize(c->stream));
    if (!h[2]) break;
    c->feed_wcap *= 4;
  }
  c->n_word_occ += h[0];
  const uint64_t U = h[1];
  if (U) {
    YT_CUDA(c, c->wpos.reserve((U + 1) * 8));
    YT_CUDA(c, c->wfreq.reserve((U + 1) * 8));
    YT_CUDA(c, c->wlen.reserve((U + 1) * 8));
    YT_CUDA(c, c->scratch_key.reserve((U + 1) * 8));
    auto *mlen = c->wlen.as<unsigned long long>(), *moff = c->scratch_key.as<unsigned long long>();
    WordTab wt{c->wkey.as<unsigned long long>(), c->wcnt.as<unsigned long long>(), c->feed_wcap - 1};
    const unsigned grid = (unsigned)grid_for(c, U, 256, 8);
    word_compact_kernel<<<grid_for(c, c->feed_wcap, 256, 8), 256, 0, c->stream>>>(wt, counters, c->wpos.as<uint64_t>(),
                                                                                  c->wfreq.as<uint64_t>());
    WordTab ft{c->fkey.as<unsigned long long>(), c->fcnt.as<unsigned long long>(), c->feed_fcap - 1};
    word_merge_lookup_kernel<<<grid, 256, 0, c->stream>>>(d, m, c->wpos.as<uint64_t>(), c->wfreq.as<uint64_t>(), U, ft,
                                                          c->arena.as<uint8_t>() + 16, mlen, counters);
    c->launches += 2;
    if (device_scan(c, mlen, U, moff, counters + 4)) return 1;
    YT_CUDA(c, cudaMemcpyAsync(h + 4, counters + 4, 16, cudaMemcpyDeviceToHost, c->stream));
    YT_CUDA(c, cudaStreamSynchronize(c->stream));
    const uint64_t bytes = h[4], fresh = h[5];
    if (fresh) {
      if (c->arena_len + bytes >= POS_MASK) YT_FAIL(c, "fed corpus: its unique words exceed 2^40 bytes");
      if (arena_reserve(c, c->arena_len + bytes) || ftab_reserve(c, fresh)) return 1;
      ft = WordTab{c->fkey.as<unsigned long long>(), c->fcnt.as<unsigned long long>(), c->feed_fcap - 1};
      word_merge_insert_kernel<<<grid, 256, 0, c->stream>>>(d, m, c->wpos.as<uint64_t>(), c->wfreq.as<uint64_t>(), U, mlen,
                                                            moff, ft, c->arena.as<uint8_t>() + 16, c->arena_len);
      c->launches++;
      c->arena_len += bytes;
      c->feed_fn += fresh;
    }
  }
  YT_CUDA(c, cudaGetLastError());
  YT_CUDA(c, cudaEventRecord(c->ev_feed_done[s], c->stream));
  c->feed_pieces++;
  note_peak(c);
  return 0;
}

// The first `cut` bytes of the staging buffer being filled become a piece: copied now, processed after the next cut.
static int feed_submit(yttm_ctx *c, uint64_t cut) {
  const int s = c->feed_cur, o = s ^ 1;
  const uint64_t tail = c->feed_len - cut;
  YT_CUDA(c, cudaEventSynchronize(c->ev_feed_copied[o]));   // the copy of the piece before read buffer o
  if (stage_reserve(c, o, tail)) return 1;
  if (tail) std::memcpy(c->feed_stage[o], c->feed_stage[s] + cut, tail);
  if (cut > c->feed_dev[s].cap) {   // the piece buffer grows: its last piece's passes are done first
    YT_CUDA(c, cudaStreamSynchronize(c->stream));
    YT_CUDA(c, c->feed_dev[s].reserve(cut));
  }
  YT_CUDA(c, cudaStreamWaitEvent(c->stream2, c->ev_feed_done[s], 0));
  YT_CUDA(c, cudaMemcpyAsync(c->feed_dev[s].p, c->feed_stage[s], cut, cudaMemcpyHostToDevice, c->stream2));
  YT_CUDA(c, cudaEventRecord(c->ev_feed_copied[s], c->stream2));
  if (c->feed_pending >= 0 && feed_process(c, c->feed_pending, c->feed_pending_len)) return 1;
  c->feed_pending = s;
  c->feed_pending_len = cut;
  c->feed_cur = o;
  c->feed_len = c->feed_nows = tail;   // what follows the last whitespace byte holds none
  return 0;
}

int yttm_train_feed_begin(yttm_ctx *c) {
  YT_CUDA(c, cudaSetDevice(c->device));
  if (ensure_stream2(c)) return 1;
  for (int s = 0; s < 2; s++) {
    if (!c->ev_feed_copied[s]) YT_CUDA(c, cudaEventCreateWithFlags(&c->ev_feed_copied[s], cudaEventDisableTiming));
    if (!c->ev_feed_done[s]) YT_CUDA(c, cudaEventCreateWithFlags(&c->ev_feed_done[s], cudaEventDisableTiming));
  }
  // a new training starts, as in yttm_train_load_corpus; the corpus of an earlier one does not stay resident
  if (feed_release(c)) return 1;
  c->text_buf.release();
  c->d_text = nullptr;
  c->n_text = 0;
  c->text_external = false;
  c->have_alphabet = false;
  c->pipe_hist = false;
  c->pipe_wtab_cap = 0;
  c->n_words = c->n_slots = c->n_unique = c->n_word_occ = 0;
  c->pcap = 0;
  c->stats = yttm_train_stats{};
  ytc::timers_reset(c);
  c->dev_peak = 0;
  c->feed_piece = (uint64_t)ytc::env_int("YTTM_TRAIN_FEED_PIECE_KB", 32 << 10, 1, INT_MAX) << 10;
  c->feed_cur = 0;
  c->feed_len = c->feed_nows = 0;
  c->arena_len = c->n_fed = c->feed_pieces = c->feed_fn = 0;
  // per-piece table: one slot per 32 bytes (a piece's distinct words are far fewer than its words); the persistent
  // table and the arena start small and grow with the unique words
  c->feed_wcap = std::min<uint64_t>(std::max<uint64_t>(ytc::pow2ceil(c->feed_piece / 32), 1u << 10), 1ull << 26);
  c->feed_fcap = 1u << 10;
  YT_CUDA(c, c->hist.reserve((CP_LIMIT + 1) * 8));
  YT_CUDA(c, cudaMemsetAsync(c->hist.p, 0, (CP_LIMIT + 1) * 8, c->stream));
  YT_CUDA(c, c->counters.reserve(64));
  YT_CUDA(c, c->fkey.reserve(c->feed_fcap * 8));
  YT_CUDA(c, c->fcnt.reserve(c->feed_fcap * 8));
  YT_CUDA(c, cudaMemsetAsync(c->fkey.p, 0, c->feed_fcap * 8, c->stream));
  YT_CUDA(c, cudaMemsetAsync(c->fcnt.p, 0, c->feed_fcap * 8, c->stream));
  YT_CUDA(c, c->arena.reserve(1u << 16));
  YT_CUDA(c, cudaMemsetAsync(c->arena.p, ' ', 16, c->stream));
  c->feeding = true;
  note_peak(c);
  return 0;
}

int yttm_train_feed(yttm_ctx *c, const char *bytes, uint64_t n) {
  YT_CUDA(c, cudaSetDevice(c->device));
  if (!c->feeding) YT_FAIL(c, "yttm_train_feed: yttm_train_feed_begin has not run");
  c->n_fed += n;
  while (n) {
    const uint64_t room = c->feed_len < c->feed_piece ? c->feed_piece - c->feed_len : c->feed_piece;
    const uint64_t take = std::min(n, room);
    if (stage_reserve(c, c->feed_cur, c->feed_len + take)) return 1;
    std::memcpy(c->feed_stage[c->feed_cur] + c->feed_len, bytes, take);
    c->feed_len += take;
    bytes += take;
    n -= take;
    if (c->feed_len < c->feed_piece) continue;
    const uint64_t cut = piece_cut(reinterpret_cast<const char *>(c->feed_stage[c->feed_cur]) + c->feed_nows,
                                   c->feed_len - c->feed_nows);
    if (!cut) { c->feed_nows = c->feed_len; continue; }   // no whitespace byte yet: the piece grows until one comes
    if (feed_submit(c, c->feed_nows + cut)) return 1;
  }
  return 0;
}

int yttm_train_feed_end(yttm_ctx *c, uint64_t *data_len, uint64_t *n_distinct) {
  YT_CUDA(c, cudaSetDevice(c->device));
  if (!c->feeding) YT_FAIL(c, "yttm_train_feed_end: yttm_train_feed_begin has not run");
  if (c->feed_len && feed_submit(c, c->feed_len)) return 1;   // the last piece ends with the corpus
  if (c->feed_pending >= 0 && feed_process(c, c->feed_pending, c->feed_pending_len)) return 1;
  c->feed_pending = -1;
  // the persistent table -> wpos / wfreq (arena positions); the arena with its pads becomes the text
  const uint64_t U = c->feed_fn;
  auto *counters = c->counters.as<unsigned long long>();
  YT_CUDA(c, c->wpos.reserve((U + 1) * 8));
  YT_CUDA(c, c->wfreq.reserve((U + 1) * 8));
  YT_CUDA(c, cudaMemsetAsync(counters + 3, 0, 8, c->stream));
  if (U) {
    WordTab ft{c->fkey.as<unsigned long long>(), c->fcnt.as<unsigned long long>(), c->feed_fcap - 1};
    word_compact_kernel<<<grid_for(c, c->feed_fcap, 256, 8), 256, 0, c->stream>>>(ft, counters, c->wpos.as<uint64_t>(),
                                                                                  c->wfreq.as<uint64_t>());
    c->launches++;
  }
  if (arena_reserve(c, c->arena_len)) return 1;
  YT_CUDA(c, cudaMemsetAsync(c->arena.as<uint8_t>() + 16 + c->arena_len, ' ', 32, c->stream));
  YT_CUDA(c, cudaGetLastError());
  note_peak(c);
  std::swap(c->text_buf, c->arena);
  if (feed_release(c)) return 1;   // (synchronises: the compaction has run)
  c->wkey.release(); c->wcnt.release();   // the per-piece table
  c->d_text = c->text_buf.as<uint8_t>() + 16;
  c->n_text = c->arena_len;
  c->n_unique = U;
  c->fed_words = true;
  return hist_summarise(c, data_len, n_distinct);
}

static int hist_summarise(yttm_ctx *c, uint64_t *data_len, uint64_t *n_distinct) {
  std::vector<unsigned long long> h(CP_LIMIT + 1);
  YT_CUDA(c, cudaMemcpyAsync(h.data(), c->hist.p, (CP_LIMIT + 1) * 8, cudaMemcpyDeviceToHost, c->stream));
  YT_CUDA(c, cudaStreamSynchronize(c->stream));
  c->h_hist_cp.clear(); c->h_hist_cnt.clear();
  for (uint32_t cp = 0; cp < CP_LIMIT; cp++)
    if (h[cp]) { c->h_hist_cp.push_back(cp); c->h_hist_cnt.push_back(h[cp]); }
  c->data_len = h[CP_LIMIT];
  if (data_len) *data_len = c->data_len;
  if (n_distinct) *n_distinct = c->h_hist_cp.size();
  return 0;
}

int yttm_train_char_hist(yttm_ctx *c, uint64_t *data_len, uint64_t *n_distinct) {
  YT_CUDA(c, cudaSetDevice(c->device));
  if (c->feeding) YT_FAIL(c, "yttm_train_char_hist: yttm_train_feed_end has not run");
  if (c->fed_words) return hist_summarise(c, data_len, n_distinct);   // counted per piece (the text is the word arena)
  if (c->pipe_hist) {   // counted while the text was copied (yttm_train_load_corpus)
    c->pipe_hist = false;
    return hist_summarise(c, data_len, n_distinct);
  }
  YT_CUDA(c, c->hist.reserve((CP_LIMIT + 1) * 8));
  YT_CUDA(c, cudaMemsetAsync(c->hist.p, 0, (CP_LIMIT + 1) * 8, c->stream));
  ytc::timer_begin(c, "char_hist");
  if (c->n_text) {
    char_hist_kernel<<<grid_for(c, c->n_text / 16 + 1, 512, 4), 512, 0, c->stream>>>(c->d_text, c->n_text,
                                                                            c->hist.as<unsigned long long>());
    c->launches++;
  }
  ytc::timer_end(c, "char_hist");
  YT_CUDA(c, cudaGetLastError());
  return hist_summarise(c, data_len, n_distinct);
}

int yttm_train_char_hist_devptr(yttm_ctx *c, void **dptr, uint64_t *n_u64) {
  if (!c->hist.p) YT_FAIL(c, "char_hist not computed");
  *dptr = c->hist.p;
  *n_u64 = CP_LIMIT + 1;
  return 0;
}
int yttm_train_char_hist_refresh(yttm_ctx *c, uint64_t *data_len, uint64_t *n_distinct) {
  if (!c->hist.p) YT_FAIL(c, "char_hist not computed");
  return hist_summarise(c, data_len, n_distinct);
}

int yttm_train_get_char_hist(yttm_ctx *c, uint32_t *cps, uint64_t *counts) {
  std::memcpy(cps, c->h_hist_cp.data(), c->h_hist_cp.size() * 4);
  std::memcpy(counts, c->h_hist_cnt.data(), c->h_hist_cnt.size() * 8);
  return 0;
}

int yttm_train_set_alphabet(yttm_ctx *c, const uint32_t *cps, const uint32_t *ids, uint64_t n_kept, uint32_t space_id) {
  YT_CUDA(c, cudaSetDevice(c->device));
  std::vector<uint32_t> tab(CP_LIMIT, NO_ID);
  for (uint64_t i = 0; i < n_kept; i++) {
    if (cps[i] >= CP_LIMIT) YT_FAIL(c, "alphabet code point out of range");
    tab[cps[i]] = ids[i];
  }
  YT_CUDA(c, c->cp2id.reserve(CP_LIMIT * 4));
  YT_CUDA(c, cudaMemcpyAsync(c->cp2id.p, tab.data(), CP_LIMIT * 4, cudaMemcpyHostToDevice, c->stream));
  YT_CUDA(c, cudaStreamSynchronize(c->stream));
  c->space_id = space_id;
  c->have_alphabet = true;
  return 0;
}

static int finish_build(yttm_ctx *c, yttm_train_stats *stats) {
  ytc::timer_begin(c, "pair_hist");
  // first guess: one slot per two tokens (the distinct pairs of the corpora measured so far are 2 - 13 % of the tokens;
  // the table is accepted at load <= 1/4).  Starting at the floor and doubling cost five histogram passes on the
  // multilingual corpus (60 ms per GB); a partition is only swept by the rare refreshes of the front, so a roomy table
  // costs nothing per merge.  (YTTM_PAIR_CAP_FLOOR still forces small tables in the tests.)
  const uint64_t guess = pair_cap_floor_knob() ? 0 : c->n_slots / 2;
  int rc = rebuild_pair_table(c, std::max<uint64_t>(pair_cap_floor(), guess));
  ytc::timer_end(c, "pair_hist");
  if (rc) return rc;
  YtLoopCtl *ctl = c->ctl.as<YtLoopCtl>();
  YtLoopCtl h{};
  YT_CUDA(c, cudaMemcpyAsync(&h, ctl, sizeof(h), cudaMemcpyDeviceToHost, c->stream));
  YT_CUDA(c, cudaStreamSynchronize(c->stream));
  h.n_done = 0; h.stop = 0; h.dead = 0; h.slots = c->n_slots;
  YT_CUDA(c, cudaMemcpyAsync(ctl, &h, sizeof(h), cudaMemcpyHostToDevice, c->stream));
  YT_CUDA(c, cudaStreamSynchronize(c->stream));
  c->stats.n_bytes = c->fed_words ? c->n_fed : c->n_text;
  c->stats.n_words = c->n_word_occ;
  c->stats.n_unique = c->n_words;
  c->stats.n_tokens = c->n_slots;
  if (stats) *stats = c->stats;
  note_peak(c);
  return 0;
}

// Phase 2a: word split + dedup of the current text -> wpos / wfreq (U unique words).  list != nullptr: the text is a
// list of weighted words received from the other ranks (n_src sources, source k = words [word_off[k], word_off[k+1])
// whose positions are relative to byte_off[k]).
struct WordList { const uint64_t *pos, *freq; const uint64_t *word_off, *byte_off; uint32_t n_src; };
static int build_word_table(yttm_ctx *c, const WordList *list, uint64_t *n_unique) {
  const uint64_t n = c->n_text;
  YT_CUDA(c, c->counters.reserve(64));
  auto *counters = c->counters.as<unsigned long long>();
  ytc::timer_begin(c, list ? "word_import" : "word_count");
  const uint64_t guess = list ? list->word_off[list->n_src] * 2 + 1 : n / 16 + 1;
  uint64_t cap = std::min<uint64_t>(std::max<uint64_t>(ytc::pow2ceil(guess), 1u << 16), 1ull << 26);
  unsigned long long h_cnt[4] = {0, 0, 0, 0};
  bool piped = false;
  if (!list && c->pipe_wtab_cap) {   // built while the text was copied (yttm_train_load_corpus)
    cap = c->pipe_wtab_cap;
    c->pipe_wtab_cap = 0;
    YT_CUDA(c, cudaMemcpyAsync(h_cnt, counters, 32, cudaMemcpyDeviceToHost, c->stream));
    YT_CUDA(c, cudaStreamSynchronize(c->stream));
    if (!h_cnt[2]) piped = true;
    else cap *= 4;   // it overflowed: the plain passes below start over with a larger table
  }
  for (int attempt = 0; !piped; attempt++) {  // retry with a larger table on overflow
    if (attempt > 10) YT_FAIL(c, "word table: too many retries");
    YT_CUDA(c, c->wkey.reserve(cap * 8));
    YT_CUDA(c, c->wcnt.reserve(cap * 8));
    YT_CUDA(c, cudaMemsetAsync(c->wkey.p, 0, cap * 8, c->stream));
    YT_CUDA(c, cudaMemsetAsync(c->wcnt.p, 0, cap * 8, c->stream));
    YT_CUDA(c, cudaMemsetAsync(counters, 0, 64, c->stream));
    WordTab wt{c->wkey.as<unsigned long long>(), c->wcnt.as<unsigned long long>(), cap - 1};
    if (list) {
      for (uint32_t k = 0; k < list->n_src; k++) {
        const uint64_t w0 = list->word_off[k], nw = list->word_off[k + 1] - w0;
        if (!nw) continue;
        word_insert_list_kernel<<<grid_for(c, nw, 256, 8), 256, 0, c->stream>>>(c->d_text, n, list->byte_off[k], list->pos + w0,
                                                                              list->freq + w0, nw, wt, counters, cap / 2);
        c->launches++;
      }
    } else if (n) {
      word_insert_kernel<<<grid_for(c, n, 256, 8), 256, 0, c->stream>>>(c->d_text, n, 0, n, wt, counters, cap / 2);
      c->launches++;
    }
    YT_CUDA(c, cudaGetLastError());
    YT_CUDA(c, cudaMemcpyAsync(h_cnt, counters, 32, cudaMemcpyDeviceToHost, c->stream));
    YT_CUDA(c, cudaStreamSynchronize(c->stream));
    if (!h_cnt[2]) break;
    cap *= 4;
  }
  c->n_word_occ = h_cnt[0];
  const uint64_t U = h_cnt[1];
  YT_CUDA(c, c->wpos.reserve((U + 1) * 8));
  YT_CUDA(c, c->wfreq.reserve((U + 1) * 8));
  if (U) {
    WordTab wt{c->wkey.as<unsigned long long>(), c->wcnt.as<unsigned long long>(), cap - 1};
    word_compact_kernel<<<grid_for(c, cap, 256, 8), 256, 0, c->stream>>>(wt, counters, c->wpos.as<uint64_t>(),
                                                                         c->wfreq.as<uint64_t>());
    c->launches++;
  }
  ytc::timer_end(c, list ? "word_import" : "word_count");
  YT_CUDA(c, cudaGetLastError());
  *n_unique = U;
  c->n_unique = U;
  return 0;
}

// Phase 2b + 3: tokenise the U unique words (wpos / wfreq) into the packed buffer, build the pair table.
static int build_tokens(yttm_ctx *c, uint64_t U, yttm_train_stats *stats) {
  const uint64_t n = c->n_text;
  auto *counters = c->counters.as<unsigned long long>();
  ytc::timer_begin(c, "tokenise");
  YT_CUDA(c, c->wlen.reserve((U + 1) * 8));
  ytc::DevBuf &scanb = c->scratch_key;
  YT_CUDA(c, scanb.reserve((U + 1) * 8));
  auto *lens = c->wlen.as<unsigned long long>();
  auto *scan = scanb.as<unsigned long long>();
  unsigned long long T = 0;
  c->cur = 0;
  YT_CUDA(c, c->off[0].reserve((U + 2) * 4));
  if (U) {
    unsigned nb = (unsigned)((U + 255) / 256);
    word_tokens_kernel<0><<<nb, 256, 0, c->stream>>>(c->d_text, n, c->wpos.as<uint64_t>(), U, c->cp2id.as<uint32_t>(),
                                                     c->space_id, lens, nullptr, nullptr, nullptr);
    c->launches++;
    unsigned long long too_many = 0;
    if (c->fed_words) {   // a fed corpus is not bounded by 2^40 bytes, so neither is a word's count change
      YT_CUDA(c, cudaMemsetAsync(counters + 5, 0, 8, c->stream));
      word_count_limit_kernel<<<nb, 256, 0, c->stream>>>(lens, c->wfreq.as<uint64_t>(), U, counters + 5);
      c->launches++;
      YT_CUDA(c, cudaMemcpyAsync(&too_many, counters + 5, 8, cudaMemcpyDeviceToHost, c->stream));
    }
    if (device_scan(c, lens, U, scan, counters + 4)) return 1;
    YT_CUDA(c, cudaMemcpyAsync(&T, counters + 4, 8, cudaMemcpyDeviceToHost, c->stream));
    YT_CUDA(c, cudaStreamSynchronize(c->stream));
    if (too_many) YT_FAIL(c, "fed corpus: a word's frequency x tokens must stay below 2^43");
    if (T >= 0xfffffff0ull) YT_FAIL(c, "more than 2^32 tokens in the unique words of one shard");
    YT_CUDA(c, c->tok[0].reserve((T + 4) * 4));
    word_tokens_kernel<1><<<nb, 256, 0, c->stream>>>(c->d_text, n, c->wpos.as<uint64_t>(), U, c->cp2id.as<uint32_t>(),
                                                     c->space_id, lens, scan, c->tok[0].as<uint32_t>(),
                                                     c->off[0].as<uint32_t>());
    c->launches++;
  } else {
    YT_CUDA(c, cudaMemsetAsync(c->off[0].p, 0, 8, c->stream));
  }
  YT_CUDA(c, cudaGetLastError());
  // frequencies travel with the words: freq[0] aliases wfreq (swap the buffers)
  std::swap(c->freq[0], c->wfreq);
  c->n_words = U;
  c->n_slots = T;
  // drop words that vanished (only removed chars) or cannot pair; gives the canonical layout
  if (compact_words(c)) return 1;
  ytc::timer_end(c, "tokenise");
  return finish_build(c, stats);
}

int yttm_train_build(yttm_ctx *c, yttm_train_stats *stats) {
  YT_CUDA(c, cudaSetDevice(c->device));
  if (c->feeding) YT_FAIL(c, "yttm_train_build: yttm_train_feed_end has not run");
  if (!c->have_alphabet) YT_FAIL(c, "yttm_train_build: alphabet not set");
  uint64_t U = c->n_unique;   // a fed corpus: its words are in wpos / wfreq already
  if (c->fed_words) {
    if (c->pcap) YT_FAIL(c, "yttm_train_build: the fed words were built already (feed the corpus again)");
  } else if (build_word_table(c, nullptr, &U)) {
    return 1;
  }
  return build_tokens(c, U, stats);
}

// ---- multi-GPU (one process per GPU; include/yttm_b200.h has the protocol) ---------------------------------------
struct XqHandle {  // what yttm_train_dist_handle writes (128 bytes)
  uint64_t magic, pid, ptr, bytes;
  int32_t device, pad;
  cudaIpcMemHandle_t ipc;
};
static_assert(sizeof(XqHandle) <= 128, "XqHandle must fit the 128-byte slot of the C ABI");
constexpr uint64_t XQ_MAGIC = 0x3151585f4d545459ull;

int yttm_train_dist_init(yttm_ctx *c, uint32_t rank, uint32_t world, void *handle_out) {
  YT_CUDA(c, cudaSetDevice(c->device));
  if (world < 1 || world > (uint32_t)XQ_MAX_WORLD || rank >= world) YT_FAIL(c, "yttm_train_dist_init: world must be 1..8, rank < world");
  if (ensure_ctl(c)) return 1;
  YT_CUDA(c, cudaMemsetAsync(c->ctl.p, 0, sizeof(YtLoopCtl), c->stream));  // exchange rounds restart at 0 on every rank
  if (xq_alloc(c, rank, world)) return 1;
  XqHandle h{};
  h.magic = XQ_MAGIC; h.pid = (uint64_t)getpid(); h.ptr = (uint64_t)(uintptr_t)c->xq_buf.p; h.bytes = c->xq_bytes;
  h.device = c->device;
  if (world > 1) YT_CUDA(c, cudaIpcGetMemHandle(&h.ipc, c->xq_buf.p));
  std::memset(handle_out, 0, 128);
  std::memcpy(handle_out, &h, sizeof(h));
  return 0;
}

int yttm_train_dist_connect(yttm_ctx *c, const void *handles) {
  YT_CUDA(c, cudaSetDevice(c->device));
  if (!c->xq_buf.p) YT_FAIL(c, "yttm_train_dist_connect: yttm_train_dist_init has not run");
  for (uint32_t d = 0; d < c->xq_world; d++) {
    if (d == c->xq_me) continue;
    XqHandle h;
    std::memcpy(&h, static_cast<const unsigned char *>(handles) + 128 * d, sizeof(h));
    if (h.magic != XQ_MAGIC || h.bytes != c->xq_bytes) YT_FAIL(c, "yttm_train_dist_connect: bad handle (ranks disagree on the geometry?)");
    if (h.pid == (uint64_t)getpid()) {  // same process (tests, one thread per GPU): the pointer itself, peer access on
      if (h.device != c->device) {
        cudaError_t e = cudaDeviceEnablePeerAccess(h.device, 0);
        if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) YT_CUDA(c, e);
        (void)cudaGetLastError();
      }
      c->xq_peer[d] = reinterpret_cast<void *>((uintptr_t)h.ptr);
      c->xq_peer_ipc[d] = false;
    } else {
      void *p = nullptr;
      YT_CUDA(c, cudaIpcOpenMemHandle(&p, h.ipc, cudaIpcMemLazyEnablePeerAccess));
      c->xq_peer[d] = p;
      c->xq_peer_ipc[d] = true;
    }
  }
  c->xq_connected = true;
  return 0;
}

int yttm_train_dist_word_table(yttm_ctx *c, uint64_t *n_unique) {
  YT_CUDA(c, cudaSetDevice(c->device));
  return build_word_table(c, nullptr, n_unique);
}

int yttm_train_dist_export_words(yttm_ctx *c, uint64_t *bytes_per_dst, uint64_t *words_per_dst, void **d_bytes,
                                 void **d_pos, void **d_freq) {
  YT_CUDA(c, cudaSetDevice(c->device));
  const uint32_t world = c->xq_world;
  const uint64_t U = c->n_unique;
  YT_CUDA(c, c->counters.reserve(64));
  ytc::DevBuf &cur = c->scan_tmp;  // 3 x world cursors
  YT_CUDA(c, cur.reserve(3 * 8 * XQ_MAX_WORLD));
  auto *cb = cur.as<unsigned long long>(), *cw = cb + XQ_MAX_WORLD, *base = cw + XQ_MAX_WORLD;
  YT_CUDA(c, cudaMemsetAsync(cb, 0, 3 * 8 * XQ_MAX_WORLD, c->stream));
  const unsigned grid = (unsigned)grid_for(c, std::max<uint64_t>(U, 1), 256, 8);
  if (U) {
    word_export_kernel<0><<<grid, 256, 0, c->stream>>>(c->d_text, c->n_text, c->wpos.as<uint64_t>(), c->wfreq.as<uint64_t>(), U,
                                                       world, cb, cw, nullptr, nullptr, nullptr, nullptr);
    c->launches++;
  }
  unsigned long long hb[2 * XQ_MAX_WORLD];
  YT_CUDA(c, cudaMemcpyAsync(hb, cb, sizeof(hb), cudaMemcpyDeviceToHost, c->stream));
  YT_CUDA(c, cudaStreamSynchronize(c->stream));
  unsigned long long bb[XQ_MAX_WORLD], wb[XQ_MAX_WORLD], tb = 0, tw = 0;
  for (uint32_t d = 0; d < world; d++) {
    bytes_per_dst[d] = hb[d]; words_per_dst[d] = hb[XQ_MAX_WORLD + d];
    bb[d] = tb; wb[d] = tw; tb += hb[d]; tw += hb[XQ_MAX_WORLD + d];
  }
  // the export buffers reuse table scratch that the word phase no longer needs
  YT_CUDA(c, c->scratch_key.reserve(tb + 64));
  YT_CUDA(c, c->scratch_cnt.reserve((tw + 1) * 8));
  YT_CUDA(c, c->wlen.reserve((tw + 1) * 8));
  YT_CUDA(c, cudaMemcpyAsync(cb, bb, 8 * world, cudaMemcpyHostToDevice, c->stream));
  YT_CUDA(c, cudaMemcpyAsync(cw, wb, 8 * world, cudaMemcpyHostToDevice, c->stream));
  YT_CUDA(c, cudaMemcpyAsync(base, bb, 8 * world, cudaMemcpyHostToDevice, c->stream));
  if (U) {
    word_export_kernel<1><<<grid, 256, 0, c->stream>>>(c->d_text, c->n_text, c->wpos.as<uint64_t>(), c->wfreq.as<uint64_t>(), U,
                                                       world, cb, cw, base, c->scratch_key.as<uint8_t>(),
                                                       c->scratch_cnt.as<uint64_t>(), c->wlen.as<uint64_t>());
    c->launches++;
  }
  YT_CUDA(c, cudaGetLastError());
  YT_CUDA(c, cudaStreamSynchronize(c->stream));
  *d_bytes = c->scratch_key.p; *d_pos = c->scratch_cnt.p; *d_freq = c->wlen.p;
  return 0;
}

int yttm_train_dist_import_words(yttm_ctx *c, const void *d_bytes, const uint64_t *bytes_per_src, const void *d_pos,
                                 const void *d_freq, const uint64_t *words_per_src, yttm_train_stats *stats) {
  YT_CUDA(c, cudaSetDevice(c->device));
  if (!c->have_alphabet) YT_FAIL(c, "yttm_train_dist_import_words: alphabet not set");
  const uint32_t world = c->xq_world;
  uint64_t bo[XQ_MAX_WORLD + 1], wo[XQ_MAX_WORLD + 1];
  bo[0] = wo[0] = 0;
  for (uint32_t k = 0; k < world; k++) { bo[k + 1] = bo[k] + bytes_per_src[k]; wo[k + 1] = wo[k] + words_per_src[k]; }
  const uint64_t n = bo[world], nw = wo[world];
  if (n >= POS_MASK) YT_FAIL(c, "imported words too large");
  // the received words become this rank's text (its own shard is no longer needed)
  ytc::DevBuf fresh;
  YT_CUDA(c, fresh.reserve(n + 64));
  uint8_t *tb = fresh.as<uint8_t>();
  YT_CUDA(c, cudaMemsetAsync(tb, ' ', 16, c->stream));
  YT_CUDA(c, cudaMemsetAsync(tb + 16 + n, ' ', 32, c->stream));
  if (n) YT_CUDA(c, cudaMemcpyAsync(tb + 16, d_bytes, n, cudaMemcpyDeviceToDevice, c->stream));
  ytc::DevBuf lp, lf;  // private copies: the caller's buffers may be the export scratch of this context
  YT_CUDA(c, lp.reserve((nw + 1) * 8));
  YT_CUDA(c, lf.reserve((nw + 1) * 8));
  if (nw) {
    YT_CUDA(c, cudaMemcpyAsync(lp.p, d_pos, nw * 8, cudaMemcpyDeviceToDevice, c->stream));
    YT_CUDA(c, cudaMemcpyAsync(lf.p, d_freq, nw * 8, cudaMemcpyDeviceToDevice, c->stream));
  }
  YT_CUDA(c, cudaStreamSynchronize(c->stream));
  c->text_buf.release();
  c->text_buf = fresh;
  c->d_text = tb + 16;
  c->n_text = n;
  c->text_external = false;
  WordList wl{lp.as<uint64_t>(), lf.as<uint64_t>(), wo, bo, world};
  uint64_t U = 0;
  int rc = build_word_table(c, &wl, &U);
  if (!rc) rc = build_tokens(c, U, stats);
  lp.release(); lf.release();
  return rc;
}

int yttm_train_export_words(yttm_ctx *c, uint32_t *tokens, uint64_t tokens_cap, uint32_t *offsets, uint64_t *freq,
                            uint64_t words_cap, uint64_t *n_words, uint64_t *n_tokens) {
  YT_CUDA(c, cudaSetDevice(c->device));
  if (!c->pcap) YT_FAIL(c, "yttm_train_export_words: yttm_train_build has not run");
  *n_words = c->n_words;
  *n_tokens = c->n_slots;
  if (!tokens) return 0;  // size query
  if (tokens_cap < c->n_slots || words_cap < c->n_words) YT_FAIL(c, "export_words: buffers too small");
  YT_CUDA(c, cudaMemcpyAsync(tokens, c->tok[c->cur].p, c->n_slots * 4, cudaMemcpyDeviceToHost, c->stream));
  YT_CUDA(c, cudaMemcpyAsync(offsets, c->off[c->cur].p, (c->n_words + 1) * 4, cudaMemcpyDeviceToHost, c->stream));
  YT_CUDA(c, cudaMemcpyAsync(freq, c->freq[c->cur].p, c->n_words * 8, cudaMemcpyDeviceToHost, c->stream));
  YT_CUDA(c, cudaStreamSynchronize(c->stream));
  return 0;
}

int yttm_train_import_words(yttm_ctx *c, const uint32_t *tokens, uint64_t n_tokens, const uint32_t *offsets,
                            const uint64_t *freq, uint64_t n_words, yttm_train_stats *stats) {
  YT_CUDA(c, cudaSetDevice(c->device));
  if (n_tokens >= 0xfffffff0ull) YT_FAIL(c, "import_words: too many tokens");
  // a count change of the merge loop is freq x (pairs of a word) in a signed 44-bit field (xq_pack)
  for (uint64_t i = 0; i < n_words; i++) {
    const uint64_t len = offsets[i + 1] - offsets[i];
    if (len && freq[i] >= (1ull << 43) / len)
      YT_FAIL(c, "import_words: word " + std::to_string(i) + ": frequency x tokens must stay below 2^43");
  }
  c->cur = 0;
  YT_CUDA(c, c->tok[0].reserve((n_tokens + 4) * 4));
  YT_CUDA(c, c->off[0].reserve((n_words + 2) * 4));
  YT_CUDA(c, c->freq[0].reserve((n_words + 1) * 8));
  YT_CUDA(c, cudaMemcpyAsync(c->tok[0].p, tokens, n_tokens * 4, cudaMemcpyHostToDevice, c->stream));
  YT_CUDA(c, cudaMemcpyAsync(c->off[0].p, offsets, (n_words + 1) * 4, cudaMemcpyHostToDevice, c->stream));
  YT_CUDA(c, cudaMemcpyAsync(c->freq[0].p, freq, n_words * 8, cudaMemcpyHostToDevice, c->stream));
  YT_CUDA(c, cudaStreamSynchronize(c->stream));
  c->n_words = n_words;
  c->n_slots = n_tokens;
  return finish_build(c, stats);
}

int yttm_train_synth_words(yttm_ctx *c, uint64_t n_words, uint32_t len, uint32_t alphabet, uint64_t seed) {
  YT_CUDA(c, cudaSetDevice(c->device));
  uint64_t T = n_words * len;
  if (T >= 0xfffffff0ull) YT_FAIL(c, "synth_words: too many tokens");
  c->cur = 0;
  YT_CUDA(c, c->tok[0].reserve((T + 4) * 4));
  YT_CUDA(c, c->off[0].reserve((n_words + 2) * 4));
  YT_CUDA(c, c->freq[0].reserve((n_words + 1) * 8));
  synth_words_kernel<<<grid_for(c, n_words + 1, 256, 8), 256, 0, c->stream>>>(
      c->tok[0].as<uint32_t>(), c->off[0].as<uint32_t>(), c->freq[0].as<uint64_t>(), n_words, len, alphabet & 0xffffffu,
      seed, std::max<uint32_t>(1u, alphabet >> 24 ? 1u << (alphabet >> 24) : 1u));
  c->launches++;
  YT_CUDA(c, cudaGetLastError());
  YT_CUDA(c, cudaStreamSynchronize(c->stream));
  c->n_words = n_words;
  c->n_slots = T;
  c->n_word_occ = n_words;
  return finish_build(c, nullptr);
}

int yttm_train_scan_once(yttm_ctx *c, double *ms, uint64_t *algo_bytes) {
  YT_CUDA(c, cudaSetDevice(c->device));
  if (!c->pcap) YT_FAIL(c, "yttm_train_scan_once: yttm_train_build has not run");
  uint64_t cap = c->pcap;
  YT_CUDA(c, c->scratch_key.reserve(cap * 8));
  YT_CUDA(c, c->scratch_cnt.reserve(cap * 8));
  YT_CUDA(c, c->counters.reserve(64));
  YT_CUDA(c, cudaMemsetAsync(c->scratch_key.p, 0xff, cap * 8, c->stream));
  YT_CUDA(c, cudaMemsetAsync(c->scratch_cnt.p, 0, cap * 8, c->stream));
  YT_CUDA(c, cudaMemsetAsync(c->counters.p, 0, 64, c->stream));
  PairTab t;
  t.keys = c->scratch_key.as<unsigned long long>();
  t.cnts = c->scratch_cnt.as<unsigned long long>();
  t.rmask = c->p_rmask;
  t.nparts = c->p_nparts;
  t.n_keys = reinterpret_cast<uint32_t *>(c->counters.as<unsigned long long>() + 6);
  t.overflow = t.n_keys + 1;
  ytc::timer_begin(c, "scan");
  pair_hist_kernel<<<grid_for(c, c->n_words, 256, 8), 256, 0, c->stream>>>(
      c->tok[c->cur].as<uint32_t>(), c->off[c->cur].as<uint32_t>(), c->freq[c->cur].as<uint64_t>(), c->n_words, t);
  c->launches++;
  ytc::timer_end(c, "scan");
  YT_CUDA(c, cudaGetLastError());
  if (ms) *ms = ytc::timer_ms(c, "scan");
  if (algo_bytes) *algo_bytes = 4 * c->n_slots + 12 * c->n_words;
  return 0;
}

int yttm_train_dump_pairs(yttm_ctx *c, uint64_t *keys, uint64_t *counts, uint64_t cap, uint64_t *n) {
  YT_CUDA(c, cudaSetDevice(c->device));
  *n = 0;
  if (!c->pcap) YT_FAIL(c, "yttm_train_dump_pairs: yttm_train_build has not run");
  ytc::DevBuf dk, dc;
  YT_CUDA(c, dk.reserve((cap + 1) * 8));
  YT_CUDA(c, dc.reserve((cap + 1) * 8));
  YT_CUDA(c, c->counters.reserve(64));
  auto *cursor = c->counters.as<unsigned long long>() + 5;
  YT_CUDA(c, cudaMemsetAsync(cursor, 0, 8, c->stream));
  pair_dump_kernel<<<grid_for(c, c->pcap, 256, 8), 256, 0, c->stream>>>(
      c->pkey.as<unsigned long long>(), c->pcnt.as<unsigned long long>(), c->pcap, cursor, cap,
      dk.as<unsigned long long>(), dc.as<unsigned long long>());
  c->launches++;
  unsigned long long cnt = 0;
  YT_CUDA(c, cudaMemcpyAsync(&cnt, cursor, 8, cudaMemcpyDeviceToHost, c->stream));
  YT_CUDA(c, cudaStreamSynchronize(c->stream));
  *n = cnt;
  uint64_t m = std::min<uint64_t>(cnt, cap);
  if (m) {
    YT_CUDA(c, cudaMemcpy(keys, dk.p, m * 8, cudaMemcpyDeviceToHost));
    YT_CUDA(c, cudaMemcpy(counts, dc.p, m * 8, cudaMemcpyDeviceToHost));
  }
  dk.release(); dc.release();
  return 0;
}

int yttm_train_run(yttm_ctx *c, uint32_t first_new_id, uint32_t max_merges, uint32_t *rules_xyz, uint64_t *freqs,
                   uint32_t *n_done_out) {
  YT_CUDA(c, cudaSetDevice(c->device));
  if (!c->pcap) YT_FAIL(c, "yttm_train_run: yttm_train_build has not run");
  *n_done_out = 0;
  c->loop_relaunches = 0;
  if (max_merges == 0) return 0;
  if (ensure_loop_geometry(c)) return 1;
  YT_CUDA(c, c->frontbuf.reserve(front_buf_words((uint32_t)c->loop_blocks) * 8));  // gather buffer of the front refreshes
  if (first_new_id + (uint64_t)max_merges >= BB_ID_LIMIT) YT_FAIL(c, "yttm_train_run: token ids beyond 2^22 are not supported by the merge loop");
  YT_CUDA(c, c->d_rules.reserve((size_t)max_merges * 12 + 16));
  YT_CUDA(c, c->d_rfreq.reserve((size_t)max_merges * 8 + 16));
  YtLoopCtl *ctl = c->ctl.as<YtLoopCtl>();
  YtLoopCtl h{};
  YT_CUDA(c, cudaMemcpyAsync(&h, ctl, sizeof(h), cudaMemcpyDeviceToHost, c->stream));
  YT_CUDA(c, cudaStreamSynchronize(c->stream));
  h.n_done = 0; h.stop = 0; h.stop_why = 0; h.iters = 0; h.n_sweeps = 0;
  for (int i = 0; i < 4; i++) h.t_phase[i] = 0;
  YT_CUDA(c, cudaMemcpyAsync(ctl, &h, sizeof(h), cudaMemcpyHostToDevice, c->stream));
  // compact the words and rebuild the table from them: the counts are stale (reason & 2: lost count changes), a
  // partition ran full (reason & 4: grow) or is over the load limit (reason & 1)
  auto rebuild = [&](uint32_t reason) -> int {
    if (compact_words(c)) return 1;
    const uint32_t keep_done = h.n_done;
    // dead keys vanish in the rebuild, so the table usually keeps its size; it grows when a partition filled up
    const uint64_t want = (reason & 4u) ? c->pcap * 2 : c->pcap / 2;
    if (rebuild_pair_table(c, std::max<uint64_t>(want, pair_cap_floor()))) return 1;
    YT_CUDA(c, cudaMemcpyAsync(&h, ctl, sizeof(h), cudaMemcpyDeviceToHost, c->stream));
    YT_CUDA(c, cudaStreamSynchronize(c->stream));
    h.n_done = keep_done;
    return 0;
  };
  ytc::timer_begin(c, "merge_loop");
  while (h.n_done < max_merges && h.stop != 1) {
    LoopArgs a{};
    if (plan_tiles(c, &a)) return 1;
    if (xq_args(c, &a)) return 1;
    a.tok = c->tok[c->cur].as<uint32_t>();
    a.off = c->off[c->cur].as<uint32_t>();
    a.freq = c->freq[c->cur].as<uint64_t>();
    a.n_words = c->n_words;
    a.tab = tab_of(c);
    a.ctl = ctl;
    a.frontbuf = c->frontbuf.as<unsigned long long>();
    a.rules = c->d_rules.as<uint32_t>();
    a.rfreq = c->d_rfreq.as<unsigned long long>();
    a.first_new_id = first_new_id;
    a.max_total = max_merges;
    a.max_iters = max_merges;
    a.part_limit = (uint32_t)(((uint64_t)c->p_rmask + 1) * pair_max_load_pct() / 100);  // rebuild above this partition load (default 1/2)
    a.front_top = (uint32_t)ytc::env_int("YTTM_FRONT_TOP", 4, 1, FRONT_TOP);   // smaller front: shorter probes and scans, but more refreshes
    {  // as many places per segment as ONE trip of the drain's items holds (1 GPU: all 7; 8 GPUs: 1)
      const uint32_t nseg = c->xq_world * c->xq_nblocks;
      const uint32_t places = std::max<uint32_t>(1, std::min<uint32_t>(XQ_BOX, (uint32_t)DRAIN_ITEMS * (uint32_t)c->loop_threads / std::max<uint32_t>(nseg, 1)));
      a.drain_places = (uint32_t)ytc::env_int("YTTM_DRAIN_PLACES", (int)places, 1, XQ_BOX);
    }
    a.newp_limit = (uint32_t)ytc::env_int("YTTM_NEWP_LIMIT", (int)NEWP_LIMIT, 1, (int)NEWP_LIMIT);
    a.dead_min_slots = 4096;
    YT_CUDA(c, cudaMemsetAsync(c->frontbuf.p, 0, front_buf_words((uint32_t)c->loop_blocks) * 8, c->stream));  // refresh numbers restart at 1
#ifndef YT_SIMT_EMU
    void *args[] = {&a};
    YT_CUDA(c, cudaLaunchCooperativeKernel((void *)merge_loop_kernel, dim3(c->loop_blocks), dim3(c->loop_threads), args,
                                           (size_t)c->loop_smem, c->stream));
#else  // tests/emul/simt: every block on its own OS thread, grid.sync() = pthread barrier
    emu::launch_cooperative((unsigned)c->loop_blocks, (unsigned)c->loop_threads, (size_t)c->loop_smem,
                            [=]() { merge_loop_kernel(a); });
#endif
    c->launches++;
    YT_CUDA(c, cudaMemcpyAsync(&h, ctl, sizeof(h), cudaMemcpyDeviceToHost, c->stream));
    YT_CUDA(c, cudaStreamSynchronize(c->stream));
    c->loop_relaunches++;
    if (h.stop == 1 || h.n_done >= max_merges) {
      // The last merge of the call may have lost count changes (or an update of a full partition): the kernel reports
      // that at its exit check as stop_why, behind "done".  Rebuild now, so that the table this call leaves behind
      // (yttm_train_dump_pairs, the next yttm_train_run) is exact.
      if (h.stop_why & 6u) {
        const uint32_t keep_stop = h.stop;
        if (rebuild(h.stop_why)) return 1;
        h.stop = keep_stop; h.stop_why = 0; h.overflow = 0; h.dead = 0; h.slots = c->n_slots;
        YT_CUDA(c, cudaMemcpyAsync(ctl, &h, sizeof(h), cudaMemcpyHostToDevice, c->stream));
      }
      break;
    }
    if (h.stop != 2 && h.stop != 3) YT_FAIL(c, "merge loop left without a reason (internal error)");
    // stop == 3: compaction wanted (by some rank); stop == 2: the table wants a rebuild.  Every rank of a job
    // leaves at the same merge for the same reason (merge_loop.cuh), so the steps below run in lockstep.
    if (h.stop == 2) {
      if (rebuild(h.stop_why)) return 1;
    } else if (compact_words(c)) {
      return 1;
    }
    h.stop = 0; h.stop_why = 0; h.overflow = 0; h.dead = 0; h.slots = c->n_slots;
    YT_CUDA(c, cudaMemcpyAsync(ctl, &h, sizeof(h), cudaMemcpyHostToDevice, c->stream));
  }
  ytc::timer_end(c, "merge_loop");
  for (int i = 0; i < 4; i++) c->loop_phase_ms[i] = (double)h.t_phase[i] * 1e-6;
  c->loop_iters = h.iters;
  c->loop_sweeps = h.n_sweeps;
  c->loop_xq_round = h.xq_round;
  note_peak(c);
  *n_done_out = h.n_done;
  if (h.n_done) {
    YT_CUDA(c, cudaMemcpyAsync(rules_xyz, c->d_rules.p, (size_t)h.n_done * 12, cudaMemcpyDeviceToHost, c->stream));
    if (freqs) YT_CUDA(c, cudaMemcpyAsync(freqs, c->d_rfreq.p, (size_t)h.n_done * 8, cudaMemcpyDeviceToHost, c->stream));
    YT_CUDA(c, cudaStreamSynchronize(c->stream));
  }
  return 0;
}

}  // extern "C"
