// encode.cu — hot path (b): batch encode_as_ids on one H100.
//
// Replaces BaseEncoder::encode_parallel / encode_sentence (youtokentome/cpp/bpe.cpp:1697-1738,
// 1455-1632) behind yttm_enc_run* of include/yttm_b200.h.  The reference gives each CPU thread a
// contiguous range of sentences and runs a heap-driven merge loop per word.  Here the batch is
// one flat byte buffer in HBM and the unit of parallel work is the WORD:
//   find_words_vec_kernel       warp per 4 sentences: word starts (on raw bytes, see bpe_core.cuh) go to a global
//                               work list in byte order; every sentence records its range of work items
//   dropout = 0 (the ids of a word are a function of its bytes, so every distinct word is encoded once):
//     dedup_words_kernel        elects one representative occurrence per distinct word
//     encode_rep_words_kernel   one thread per representative: UTF-8 decode -> char ids (unknown runs collapse to
//                               one pseudo token, bpe.cpp:1513-1533) -> min-rank merge loop, leftmost first
//                               (MergeEvent2::operator< bpe.cpp:1475-1478)
//     encode_long_words_kernel  one block per representative of more than LONG_W slots
//   dropout > 0 (every occurrence draws for itself):
//     encode_words_kernel       one thread per occurrence, the same merge loop with BPE-dropout (DropoutQueue
//                               bpe.cpp:1417-1453 with a counter-based generator)
//   sentence_ids_kernel         ids per sentence; an exclusive scan turns them into output offsets
//   emit_ids_kernel             warp per sentence: copies the ids of its words into the packed output
// The ids of a word are kept in its private slots of a scratch buffer (a word of k bytes owns k+1 slots), at a
// position that is a pure function of its byte position, so no kernel depends on another block's progress.
#include <algorithm>
#include <cstdlib>
#include <cstring>

#include "common.cuh"
#include "enc_state.cuh"

using namespace yt;

namespace {

constexpr uint32_t NO_RANK = 0xffffffffu;

struct RuleTab {       // (x,y) -> (rank, z); 16 B per slot, one 128-bit load per probe
  const uint4 *slots;  // .x = x, .y = y, .z = rank, .w = z ; x == 0xffffffff => empty
  uint32_t mask;
};

__device__ __forceinline__ uint32_t rule_rank(const RuleTab &rt, uint32_t a, uint32_t b, uint32_t *z) {
  if ((a | b) & UNK_FLAG) return NO_RANK;
  uint32_t h = rule_hash(a, b) & rt.mask;
  while (true) {
    uint4 s = __ldg(rt.slots + h);
    if (s.x == a && s.y == b) { *z = s.w; return s.z; }
    if (s.x == 0xffffffffu) return NO_RANK;
    h = (h + 1) & rt.mask;
  }
}

struct EncArgs {
  const uint8_t *bytes;      // batch bytes; sentence i = [offs[i]-offs[0], offs[i+1]-offs[0])
  const uint64_t *offs;      // n_sent + 1
  uint64_t n_sent;
  int32_t *slots;            // n_bytes + 3 * n_sent
  uint32_t *ranks;           // same size: cached pair ranks of the word being merged
  uint32_t *aux;             // 6x that size, BPE-dropout only: linked list + stale events of the word
  uint32_t *word_pos;        // work list: byte position of the word start (relative to the batch)
  uint32_t *word_sent;       //            sentence index inside the batch
  unsigned long long *n_words;
  unsigned long long *n_ids;  // per sentence (uint64 so the generic scan applies)
  uint32_t *sent_wbase;       // first work item / number of work items of every sentence
  uint32_t *sent_wcnt;
  uint32_t *n_tok;            // per encoded work item (every representative, or every word with dropout): number of ids
  const uint32_t *cp2id;
  RuleTab rt;
  uint32_t space_id;
  int32_t unk_id, bos_id, eos_id;
  int bos, eos, reverse;
  uint64_t drop_thresh, seed, first_sentence;
};

// slot of the char token of batch byte p in sentence s (its word's "▁" sits one slot before the
// word's first byte): base(s) = start(s) + 3 s ; the tokens of the sentence's words sit at
// [base + 1 + rel ..], the slots base and base + len + 2 stay unused.
__device__ __forceinline__ uint64_t sent_base(uint64_t start, uint64_t s) { return start + 3 * s; }

// Word starts, FIND_SPW sentences per warp and round.  Pass 1 counts the word starts of each sentence, one atomicAdd
// per BLOCK and round reserves a contiguous range of the work list (a single counter hammered once per warp was a
// bottleneck), pass 2 writes the entries in byte order and every sentence's range of work items.  A lane owns FOUR
// consecutive bytes - one aligned 32-bit load - and decides the word starts on a 12-byte register window (previous /
// own / next word, the neighbours' by shuffle); the 4-bit flags of the first FIND_VEC_CACHE / FIND_SPW 128-byte chunks
// of every sentence stay in one register for the write pass.  word_start_at(p) == space_before(p) && !space_at(p) on
// raw bytes (a continuation byte is never a space), and the text bounds become sentinel bytes: 0x20 before the sentence
// (space_before(lo) is true; E2 96 81 cannot match across lo), 0x00 at and after its end (E2 96 81 cannot match across hi).
constexpr int FIND_VEC_CACHE = 8;
// the four bytes at batch positions p .. p+3 (p may be negative or reach past the batch), sentinels applied
__device__ __forceinline__ uint32_t find_vec_word(const uint8_t *s, int64_t p, int64_t lo, int64_t hi, int64_t n_total) {
  if (p + 4 <= lo) return 0x20202020u;
  if (p >= hi) return 0u;
  uint32_t w = 0;
  if (p >= 0 && p + 4 <= n_total) w = *reinterpret_cast<const uint32_t *>(s + p);  // p is address-aligned by construction
  else
    for (int k = 0; k < 4; k++)
      if (p + k >= 0 && p + k < n_total) w |= (uint32_t)s[p + k] << (8 * k);
  if (p < lo || p + 4 > hi)
    for (int k = 0; k < 4; k++) {
      if (p + k < lo) w = (w & ~(0xffu << (8 * k))) | (0x20u << (8 * k));
      else if (p + k >= hi) w &= ~(0xffu << (8 * k));
    }
  return w;
}
// SWAR helpers on four bytes at once: high bit of every byte that is an ASCII space (0x20 or 0x09..0x0d) / equals v
__device__ __forceinline__ uint32_t swar_eq(uint32_t w, uint32_t v4) {
  const uint32_t t = w ^ v4;
  return ~(((t & 0x7f7f7f7fu) + 0x7f7f7f7fu) | t | 0x7f7f7f7fu);
}
__device__ __forceinline__ uint32_t swar_space(uint32_t w) {
  const uint32_t b7 = w & 0x7f7f7f7fu;
  const uint32_t ge9 = b7 + 0x77777777u, ge14 = b7 + 0x72727272u;   // bit 7 of a byte: (b & 0x7f) >= 9 / >= 14 (no carry between bytes)
  return (swar_eq(w, 0x20202020u) | (ge9 & ~ge14 & ~w)) & 0x80808080u;
}
__device__ __forceinline__ uint32_t swar_mask4(uint32_t hi) {  // 0x80 bits of four bytes -> 4-bit mask
  const uint32_t m = hi >> 7;
  return (m | (m >> 7) | (m >> 14) | (m >> 21)) & 15u;
}
// word-start flags (bit k = byte p + k) of the lane's four bytes
__device__ __forceinline__ uint32_t find_vec_flags(const uint8_t *s, int64_t p, int64_t lo, int64_t hi, int64_t n_total,
                                                   unsigned lane) {
  const uint32_t c = find_vec_word(s, p, lo, hi, n_total);
  uint32_t pv = __shfl_up_sync(0xffffffffu, c, 1), nx = __shfl_down_sync(0xffffffffu, c, 1);
  if (lane == 0) pv = find_vec_word(s, p - 4, lo, hi, n_total);
  if (lane == 31) nx = find_vec_word(s, p + 4, lo, hi, n_total);
  uint32_t inside = 15u;   // bytes of this lane that belong to the sentence
  if (p < lo) inside &= lo - p >= 4 ? 0u : 15u << (uint32_t)(lo - p);
  if (p + 4 > hi) inside &= hi <= p ? 0u : 15u >> (uint32_t)(p + 4 - hi);
  if (!((swar_eq(pv, 0xe2e2e2e2u) | swar_eq(c, 0xe2e2e2e2u) | swar_eq(nx, 0xe2e2e2e2u)) & 0x80808080u)) {
    // fast path (no 0xE2 within four bytes either side, so no U+2581 can touch these positions): a word starts where an
    // ASCII space (or the sentinel in front of the sentence) is followed by a non-space byte
    const uint32_t sp = swar_mask4(swar_space(c)), sp_prev = swar_mask4(swar_space(pv)) >> 3;
    return ((sp << 1) | sp_prev) & ~sp & inside & 15u;
  }
  const uint64_t X = (uint64_t)pv | ((uint64_t)c << 32), Y = (uint64_t)c | ((uint64_t)nx << 32);  // bytes p-4 .. p+3, p .. p+7
  uint32_t f = 0;
#pragma unroll
  for (int k = 0; k < 4; k++) {
    const uint32_t t = (uint32_t)(X >> (8 * (1 + k))), u = (uint32_t)(Y >> (8 * k));  // t: bytes p+k-3 .., u: bytes p+k ..
    const bool before = is_space_byte((uint8_t)(t >> 16)) || (t & 0xffffffu) == 0x8196e2u;
    const bool at = is_space_byte((uint8_t)u) || (u & 0xffffffu) == 0x8196e2u;
    if (before && !at) f |= 1u << k;
  }
  return f & inside;
}
constexpr int FIND_SPW = 4;  // sentences per warp and round: one work-list reservation (atomic) per 32 sentences
// (at least 4 blocks per SM, the occupancy it is measured at: left free, ptxas moves the counts to local memory)
__global__ void __launch_bounds__(256, 4) find_words_vec_kernel(EncArgs a) {
  __shared__ unsigned long long s_cnt[8 * FIND_SPW], s_base;
  const unsigned lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const uint64_t o0 = a.offs[0];
  const int64_t n_total = (int64_t)(a.offs[a.n_sent] - o0);
  const int64_t mis = (int64_t)(reinterpret_cast<uintptr_t>(a.bytes) & 3u);
  constexpr uint64_t PER_ROUND = 8 * FIND_SPW;
  for (uint64_t g = (uint64_t)blockIdx.x * PER_ROUND; g < a.n_sent; g += (uint64_t)gridDim.x * PER_ROUND) {  // block-uniform
    int64_t lo[FIND_SPW], hi[FIND_SPW], start[FIND_SPW];
    uint32_t cnt[FIND_SPW];
    uint32_t cache = 0;  // flags of the first FIND_VEC_CACHE / FIND_SPW chunks of every sentence, 4 bits per chunk
    constexpr int CPS = FIND_VEC_CACHE / FIND_SPW;  // cached chunks per sentence (2: a 128-byte sentence spans at most 2)
#pragma unroll
    for (int q = 0; q < FIND_SPW; q++) {
      const uint64_t s = g + (uint64_t)wid * FIND_SPW + q;
      lo[q] = hi[q] = start[q] = 0;
      cnt[q] = 0;
      if (s < a.n_sent) {  // warp-uniform
        lo[q] = (int64_t)(a.offs[s] - o0);
        hi[q] = (int64_t)(a.offs[s + 1] - o0);
        start[q] = lo[q] - ((lo[q] + mis) & 3);  // the address of batch byte `start` is 4-byte aligned
        uint32_t mine = 0;
        int j = 0;
        for (int64_t pw = start[q]; pw < hi[q]; pw += 128, j++) {  // warp-uniform
          const uint32_t f = find_vec_flags(a.bytes, pw + 4 * lane, lo[q], hi[q], n_total, lane);
          if (j < CPS) cache |= f << (4 * (q * CPS + j));
          mine += __popc(f);
        }
        for (int o = 16; o > 0; o >>= 1) mine += __shfl_xor_sync(0xffffffffu, mine, o);
        cnt[q] = mine;
      }
      if (lane == 0) s_cnt[wid * FIND_SPW + q] = cnt[q];
    }
    __syncthreads();
    if (wid == 0) {  // exclusive prefix of the 32 sentence counts + ONE reservation for the round
      const unsigned long long c = s_cnt[lane];
      unsigned long long x = c;
      for (int o = 1; o < 32; o <<= 1) {
        const unsigned long long y = __shfl_up_sync(0xffffffffu, x, o);
        if ((int)lane >= o) x += y;
      }
      s_cnt[lane] = x - c;
      if (lane == 31) s_base = x ? atomicAdd(a.n_words, x) : 0ull;
    }
    __syncthreads();
#pragma unroll
    for (int q = 0; q < FIND_SPW; q++) {
      const uint64_t s = g + (uint64_t)wid * FIND_SPW + q;
      if (s >= a.n_sent) continue;  // warp-uniform
      unsigned long long idx = s_base + s_cnt[wid * FIND_SPW + q];
      if (lane == 0) { a.sent_wbase[s] = (uint32_t)idx; a.sent_wcnt[s] = cnt[q]; }
      if (!cnt[q]) continue;
      const unsigned below = (1u << lane) - 1u;
      int j = 0;
      for (int64_t pw = start[q]; pw < hi[q]; pw += 128, j++) {
        const int64_t p = pw + 4 * lane;
        const uint32_t f = j < CPS ? (cache >> (4 * (q * CPS + j))) & 15u : find_vec_flags(a.bytes, p, lo[q], hi[q], n_total, lane);
        const unsigned b0 = __ballot_sync(0xffffffffu, f & 1u), b1 = __ballot_sync(0xffffffffu, f & 2u),
                       b2 = __ballot_sync(0xffffffffu, f & 4u), b3 = __ballot_sync(0xffffffffu, f & 8u);
        // byte order: a lane's index = words in earlier lanes (all four bits) + its own lower bits
        const unsigned all_below = __popc(b0 & below) + __popc(b1 & below) + __popc(b2 & below) + __popc(b3 & below);
        unsigned long long i = idx + all_below;
#pragma unroll
        for (int k = 0; k < 4; k++)
          if ((f >> k) & 1u) {
            a.word_pos[i] = (uint32_t)(p + k);
            a.word_sent[i] = (uint32_t)s;
            i++;
          }
        idx += __popc(b0) + __popc(b1) + __popc(b2) + __popc(b3);
      }
    }
    __syncthreads();  // s_cnt / s_base are reused by the next round
  }
}

// Dropout > 0: one thread per word occurrence (every occurrence draws for itself).  Words of at most LOCAL_W - 1
// bytes (nearly all) are merged in thread-private local arrays (L1-resident) and only the final tokens go to the slot
// buffer; longer words work in place in their private slots in global memory.
__global__ void __launch_bounds__(128) encode_words_kernel(EncArgs a, uint64_t n_words) {
  constexpr uint32_t LOCAL_W = 40;
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  const uint64_t o0 = a.offs[0];
  const RuleTab rt = a.rt;
  auto rank = [&](uint32_t x, uint32_t y, uint32_t *z) { return rule_rank(rt, x, y, z); };
  for (uint64_t w = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; w < n_words; w += stride) {
    const uint64_t p0 = a.word_pos[w], s = a.word_sent[w];
    const uint64_t lo = a.offs[s] - o0, hi = a.offs[s + 1] - o0;
    const uint64_t slot0 = sent_base(lo, s) + 1 + (p0 - lo);
    int32_t *t = a.slots + slot0;  // k+1 private slots
    uint64_t q = p0;
    uint32_t l;
    while (q < hi && !space_at(a.bytes, q, hi, &l)) q++;
    uint32_t owned = (uint32_t)(q - p0) + 1, n;
    if (owned <= LOCAL_W) {
      int32_t lt[LOCAL_W];
      uint32_t lr[LOCAL_W];
      uint32_t laux[6 * LOCAL_W];
      // (caching z beside the ranks, or a z-by-rank table, both measured slower than re-probing the
      // L1-hot slot at merge time: 3.8 ms vs 5.8 / 4.8 ms)
      n = encode_word(a.bytes, p0, lo, hi, a.cp2id, a.space_id, rank, nullptr, a.drop_thresh, a.seed,
                      a.first_sentence + s, lt, lr, laux, &owned);
      for (uint32_t i = 0; i < n; i++) t[i] = ((uint32_t)lt[i] & UNK_FLAG) ? a.unk_id : lt[i];
    } else {
      n = encode_word(a.bytes, p0, lo, hi, a.cp2id, a.space_id, rank, nullptr, a.drop_thresh, a.seed,
                      a.first_sentence + s, t, a.ranks + slot0, a.aux + 6 * slot0, &owned);
      for (uint32_t i = 0; i < n; i++)
        if ((uint32_t)t[i] & UNK_FLAG) t[i] = a.unk_id;
    }
    a.n_tok[w] = n;
  }
}

// Words of more than LONG_W slots.  One thread merges a word in O(n^2) (min scan + shift per merge): fine for words,
// hopeless for a 100 KB "word" (a base64 blob, a URL list without blanks) - the reference's heap is O(n log n) there.
// Without dropout, encode_rep_words_kernel sets such representatives aside in a list and encode_long_words_kernel
// gives each of them a whole block.  With dropout they stay on the sequential path: the per-event draws are order
// dependent.
constexpr uint32_t LONG_W = 512;
constexpr uint32_t DEAD_T = 0xfffffffeu;  // token merged away in the current pass (has UNK_FLAG set: never a rule operand)
struct LongList {
  uint32_t *pos, *sent, *end;  // word start, sentence, word end (batch byte positions)
  uint32_t *item;              // the work item (representative) the word belongs to
  unsigned long long *n;
  uint32_t cap;                // entries; a representative that finds the list full stays on the one-thread path
};

// One block per long word, dropout = 0.  The merge order of encode_sentence (minimum rule index, leftmost first,
// bpe.cpp:1475-1478) is reproduced pass by pass: find the minimum rank r* over the word; every occurrence of that rule
// is applied in this pass, left to right without overlap - the sequential order would pick exactly these, because the
// tokens a merge creates only form pairs of HIGHER rule index (the product of rule k appears in rules > k only) and
// occurrences of the pair itself can only disappear (runs x x x ... take every second one from the run's start).
// Then the word is compacted and the ranks next to the new tokens are looked up again.  Work per pass is O(n / threads).
constexpr int LONG_T = 512;
__device__ __forceinline__ uint32_t long_block_min(uint32_t v, uint32_t *s_red) {
  for (int o = 16; o > 0; o >>= 1) v = min(v, __shfl_xor_sync(0xffffffffu, v, o));
  __syncthreads();
  if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = v;
  __syncthreads();
  uint32_t r = s_red[0];
  for (unsigned i = 1; i < (blockDim.x >> 5); i++) r = min(r, s_red[i]);
  return r;
}
// exclusive sum and inclusive max of one value per thread over the block; *tot = block sum / block max
__device__ __forceinline__ uint32_t long_block_scan_sum(uint32_t v, uint32_t *s_red, uint32_t *tot) {
  const unsigned lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
  uint32_t x = v;
  for (int o = 1; o < 32; o <<= 1) { const uint32_t y = __shfl_up_sync(0xffffffffu, x, o); if ((int)lane >= o) x += y; }
  __syncthreads();
  if (lane == 31) s_red[wid] = x;
  __syncthreads();
  uint32_t base = 0, all = 0;
  for (unsigned i = 0; i < nw; i++) { const uint32_t w = s_red[i]; if (i < wid) base += w; all += w; }
  *tot = all;
  return base + x - v;
}
__device__ __forceinline__ uint32_t long_block_scan_max(uint32_t v, uint32_t *s_red) {
  const unsigned lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  uint32_t x = v;
  for (int o = 1; o < 32; o <<= 1) { const uint32_t y = __shfl_up_sync(0xffffffffu, x, o); if ((int)lane >= o) x = max(x, y); }
  __syncthreads();
  if (lane == 31) s_red[wid] = x;
  __syncthreads();
  for (unsigned i = 0; i < wid; i++) x = max(x, s_red[i]);
  return x;
}

__global__ void __launch_bounds__(LONG_T) encode_long_words_kernel(EncArgs a, LongList ll) {
  __shared__ uint32_t s_red[LONG_T / 32];
  __shared__ uint32_t s_n, s_hit, s_z, s_xeqy;
  const uint64_t o0 = a.offs[0];
  const RuleTab rt = a.rt;
  const unsigned long long n_long = min(*ll.n, (unsigned long long)ll.cap);
  for (unsigned long long w = blockIdx.x; w < n_long; w += gridDim.x) {  // block-uniform
    const uint64_t p0 = ll.pos[w], s = ll.sent[w], q_end = ll.end[w];
    const uint64_t lo = a.offs[s] - o0, hi = a.offs[s + 1] - o0;
    const uint64_t slot0 = sent_base(lo, s) + 1 + (p0 - lo);
    uint32_t *t = reinterpret_cast<uint32_t *>(a.slots + slot0);
    uint32_t *r = a.ranks + slot0;
    if (threadIdx.x == 0) {  // decode: O(bytes), the cheap part (same rules as encode_word)
      uint32_t n = 1, l;
      bool last_unk = false;
      uint64_t q = p0;
      while (q < q_end) {
        const uint32_t cp = decode_unit(a.bytes, q, hi, &l);
        q += l;
        if (cp == INVALID_CP) continue;
        const uint32_t id = a.cp2id[cp];
        if (id == NO_ID) {
          if (!last_unk) t[n++] = UNK_FLAG | 1u;
          last_unk = true;
        } else { t[n++] = id; last_unk = false; }
      }
      t[0] = a.space_id;
      s_n = n;
    }
    __syncthreads();
    uint32_t n = s_n;
    const bool no_unit = n == 1;  // a word without a valid unit does not exist for the reference
    if (n > 1) {
      for (uint32_t i = threadIdx.x; i < n; i += LONG_T) {
        uint32_t z;
        r[i] = i + 1 < n ? rule_rank(rt, t[i], t[i + 1], &z) : NO_RANK;
      }
      __syncthreads();
      while (n > 1) {
        // ---- minimum rank of the word and one of its positions
        uint32_t best = NO_RANK, where = 0;
        for (uint32_t i = threadIdx.x; i + 1 < n; i += LONG_T)
          if (r[i] < best) { best = r[i]; where = i; }
        const uint32_t rmin = long_block_min(best, s_red);
        if (rmin == NO_RANK) break;
        if (threadIdx.x == 0) s_hit = 0xffffffffu;
        __syncthreads();
        if (best == rmin) atomicMin(&s_hit, where);  // any of them would do; the minimum is race-free
        __syncthreads();
        if (threadIdx.x == 0) {
          const uint32_t x = t[s_hit], y = t[s_hit + 1];
          uint32_t z = 0;
          rule_rank(rt, x, y, &z);
          s_z = z;
          s_xeqy = x == y;
        }
        __syncthreads();
        const uint32_t z = s_z;
        const bool xeqy = s_xeqy != 0;
        // ---- apply every occurrence, left to right without overlap (only r is read here, only t written)
        uint32_t carry = 0;  // run start + 1 of a run of hits that reaches the end of the previous chunk
        for (uint32_t b = 0; b + 1 < n; b += LONG_T) {
          const uint32_t i = b + threadIdx.x;
          const bool hit = i + 1 < n && r[i] == rmin;
          bool take = hit;
          if (xeqy) {  // x x x x ...: every second occurrence, counted from the start of the run of hits
            const bool starts = hit && !(i > 0 && r[i - 1] == rmin);
            uint32_t m = long_block_scan_max(starts ? i + 1 : 0u, s_red);
            if (m == 0) m = carry;  // the run began in an earlier chunk
            take = hit && (((i + 1 - m) & 1u) == 0);
            // hand the run start over if the last position of this chunk is still inside a run
            __syncthreads();
            if (threadIdx.x == LONG_T - 1) s_red[0] = hit ? m : 0u;
            __syncthreads();
            carry = s_red[0];
          }
          if (take) { t[i] = z; t[i + 1] = DEAD_T; }
        }
        __syncthreads();
        // ---- compact tokens and ranks (writes trail reads: destination <= source, chunk by chunk)
        uint32_t off = 0;
        for (uint32_t b = 0; b < n; b += LONG_T) {
          const uint32_t i = b + threadIdx.x;
          const uint32_t ti = i < n ? t[i] : DEAD_T, ri = i < n ? r[i] : NO_RANK;
          const uint32_t alive = ti != DEAD_T ? 1u : 0u;
          uint32_t tot;
          const uint32_t pos = long_block_scan_sum(alive, s_red, &tot);  // has the barriers between reads and writes
          if (alive) { t[off + pos] = ti; r[off + pos] = ri; }
          off += tot;
          __syncthreads();
        }
        n = off;
        // ---- ranks next to the new tokens
        for (uint32_t j = threadIdx.x; j < n; j += LONG_T) {
          if (j + 1 >= n) { r[j] = NO_RANK; continue; }
          const uint32_t u = t[j], v = t[j + 1];
          if (u == z || v == z) { uint32_t zz; r[j] = rule_rank(rt, u, v, &zz); }
        }
        __syncthreads();
      }
    }
    // ---- the reference's id-0 quirk (drop_unmerged_space0): a never-merged "▁" with id 0 leaves the output
    if (!no_unit && a.space_id == 0) {
      const bool drop = t[0] == 0;  // block-uniform (one value read by everyone)
      __syncthreads();
      if (drop) {
        for (uint32_t b0 = 0; b0 + 1 < n; b0 += LONG_T) {  // chunk by chunk: reads before writes, destination < source
          const uint32_t i = b0 + threadIdx.x;
          const uint32_t v = i + 1 < n ? t[i + 1] : 0u;
          __syncthreads();
          if (i + 1 < n) t[i] = v;
          __syncthreads();
        }
        n -= 1;
      }
    }
    // ---- final ids
    const uint32_t n_out = no_unit ? 0 : n;
    for (uint32_t i = threadIdx.x; i < n_out; i += LONG_T) {
      const uint32_t v = t[i];
      t[i] = (v & UNK_FLAG) ? (uint32_t)a.unk_id : v;
    }
    if (threadIdx.x == 0) a.n_tok[ll.item[w]] = n_out;
    __syncthreads();
  }
}

// Dropout = 0: every distinct word of the batch is encoded ONCE.  Without dropout the ids of a word are a pure function
// of its bytes [p0, q): a lead byte whose announced length reaches past q sees either the end of the sentence or the
// first byte of a space unit (never a continuation byte), INVALID_CP with length 1 in both cases (decode_unit), so
// nothing outside the word enters.  Natural text repeats its words (the bench batch: 20 M occurrences of < 200 k
// words), and the merge loop of encode_word is the expensive part of encoding a word.  Three launches:
//   dedup_words_kernel       one thread per occurrence: end of the word + 64-bit FNV-1a/mix64 hash of its bytes; an
//                            open-addressed table of (32-bit tag, work item) words, small enough to stay in L2, elects
//                            the first occurrence that claims a slot as the word's representative; later occurrences
//                            with the same tag compare BYTES with it (exactness never rests on the hash).  A word that
//                            finds neither itself nor a free slot within DEDUP_PROBES probes represents itself, so the
//                            table is a bounded cache, not a limit.
//   encode_rep_words_kernel  the per-word body, over the representatives only (list length read on the device);
//                            representatives of more than LONG_W slots go to the list of encode_long_words_kernel
//   encode_long_words_kernel a block per long representative
// emit_ids_kernel then copies the ids of a representative to every occurrence.  The slot of the first token of work
// item w is word_pos[w] + 3 word_sent[w] + 1 (sent_base(): the sentence start cancels), so a copy needs no sentence
// offsets.
constexpr unsigned long long DEDUP_EMPTY = ~0ull;
constexpr uint32_t DEDUP_PROBES = 8;
struct DedupArgs {
  unsigned long long *tab;     // (tag << 32) | representative work item ; DEDUP_EMPTY = free
  uint32_t mask;
  uint32_t *rep;               // per work item: its representative (itself if it is one)
  uint32_t *list;              // the representatives, in arrival order
  unsigned long long *n_list;
  uint32_t weak_tag;           // tests only: all tags equal, so every probe ends in the byte compare
};

__global__ void __launch_bounds__(128) dedup_words_kernel(EncArgs a, uint64_t n_words, DedupArgs d) {
  const unsigned lane = threadIdx.x & 31;
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  const uint64_t o0 = a.offs[0];
  for (uint64_t w0 = (uint64_t)blockIdx.x * blockDim.x + (threadIdx.x & ~31u); w0 < n_words; w0 += stride) {  // warp-uniform
    const uint64_t w = w0 + lane;
    bool is_rep = false;
    if (w < n_words) {
      const uint64_t p0 = a.word_pos[w], hi = a.offs[(uint64_t)a.word_sent[w] + 1] - o0;
      uint64_t q = p0, h = 0xcbf29ce484222325ull;
      uint32_t l;
      while (q < hi && !space_at(a.bytes, q, hi, &l)) { h = (h ^ a.bytes[q]) * 0x100000001b3ull; q++; }
      const uint64_t len = q - p0;
      h = mix64(h);
      const uint32_t tag = d.weak_tag ? 7u : (uint32_t)(h >> 32);
      const unsigned long long mine = ((unsigned long long)tag << 32) | (uint32_t)w;
      uint32_t idx = (uint32_t)h & d.mask, r = (uint32_t)w;
      is_rep = true;  // also the outcome of running out of probes
      for (uint32_t k = 0; k < DEDUP_PROBES; k++, idx = (idx + 1) & d.mask) {
        unsigned long long cur = *(volatile unsigned long long *)(d.tab + idx);
        if (cur == DEDUP_EMPTY) {
          cur = atomicCAS(d.tab + idx, DEDUP_EMPTY, mine);
          if (cur == DEDUP_EMPTY) break;  // slot claimed: this occurrence represents the word
        }
        if ((uint32_t)(cur >> 32) != tag) continue;
        const uint32_t w2 = (uint32_t)cur;  // written by find_words (the previous launch), like everything read below
        const uint64_t p2 = a.word_pos[w2], hi2 = a.offs[(uint64_t)a.word_sent[w2] + 1] - o0;
        // Equal iff the len bytes match AND the word at p2 ends right after them.  No space unit can start inside the
        // matching bytes: an ASCII space or a whole E2 96 81 there would be one in this word too, and an E2 96 81 that
        // starts inside and ends beyond leaves a continuation byte at p2 + len, which the end check rejects.
        bool same = true;
        for (uint64_t i = 0; i < len; i++)
          if (p2 + i >= hi2 || a.bytes[p2 + i] != a.bytes[p0 + i]) { same = false; break; }
        if (same && p2 + len < hi2 && !space_at(a.bytes, p2 + len, hi2, &l)) same = false;  // the other word is longer
        if (same) { r = w2; is_rep = false; break; }
      }
      d.rep[w] = r;
    }
    const unsigned m = __ballot_sync(0xffffffffu, is_rep);
    if (m) {  // one atomicAdd per warp reserves the list entries of its new representatives
      unsigned long long base = 0;
      if (lane == 0) base = atomicAdd(d.n_list, (unsigned long long)__popc(m));
      base = __shfl_sync(0xffffffffu, base, 0);
      if (is_rep) d.list[base + __popc(m & ((1u << lane) - 1))] = (uint32_t)w;
    }
  }
}

__global__ void __launch_bounds__(128) encode_rep_words_kernel(EncArgs a, DedupArgs d, LongList ll) {
  constexpr uint32_t LOCAL_W = 40;
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  const uint64_t o0 = a.offs[0];
  const RuleTab rt = a.rt;
  auto rank = [&](uint32_t x, uint32_t y, uint32_t *z) { return rule_rank(rt, x, y, z); };
  const unsigned long long n_list = *d.n_list;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_list; i += stride) {
    const uint32_t w = d.list[i];
    const uint64_t p0 = a.word_pos[w], s = a.word_sent[w];
    const uint64_t lo = a.offs[s] - o0, hi = a.offs[s + 1] - o0;
    const uint64_t slot0 = p0 + 3 * s + 1;
    int32_t *t = a.slots + slot0;  // k+1 private slots
    uint64_t q = p0;
    uint32_t l;
    while (q < hi && !space_at(a.bytes, q, hi, &l)) q++;
    uint32_t owned = (uint32_t)(q - p0) + 1, n;
    if (owned > LONG_W) {  // a whole block will take it (encode_long_words_kernel sets n_tok)
      const unsigned long long k = atomicAdd(ll.n, 1ull);
      if (k < ll.cap) { ll.pos[k] = (uint32_t)p0; ll.sent[k] = (uint32_t)s; ll.end[k] = (uint32_t)q; ll.item[k] = w; continue; }
    }
    if (owned <= LOCAL_W) {
      int32_t lt[LOCAL_W];
      uint32_t lr[LOCAL_W];
      n = encode_word(a.bytes, p0, lo, hi, a.cp2id, a.space_id, rank, nullptr, 0, a.seed, a.first_sentence + s, lt, lr,
                      nullptr, &owned);
      for (uint32_t k = 0; k < n; k++) t[k] = ((uint32_t)lt[k] & UNK_FLAG) ? a.unk_id : lt[k];
    } else {
      n = encode_word(a.bytes, p0, lo, hi, a.cp2id, a.space_id, rank, nullptr, 0, a.seed, a.first_sentence + s, t,
                      a.ranks + slot0, nullptr, &owned);
      for (uint32_t k = 0; k < n; k++)
        if ((uint32_t)t[k] & UNK_FLAG) t[k] = a.unk_id;
    }
    a.n_tok[w] = n;
  }
}

// ---- output ---------------------------------------------------------------------------------------------------
// The words of sentence s are the work items [sent_wbase[s], + sent_wcnt[s]) in byte order (find_words_vec_kernel); the
// ids of work item w are the n_tok[r] values at slot(word_pos[r] + 3 word_sent[r] + 1) of its representative r = rep[w]
// (r = w with dropout).  Two warp-per-sentence kernels take the ids from the encoded words straight to the packed
// output, without compacting the slot buffer:
//   sentence_ids_kernel   n_ids[s] = bos + eos + sum of n_tok over the sentence's words
//   emit_ids_kernel       every lane takes one word, a warp scan gives its place, ids are copied from the
//                         representative (reverse = mirrored index)
__global__ void __launch_bounds__(256) sentence_ids_kernel(EncArgs a, const uint32_t *__restrict__ rep) {
  const unsigned lane = threadIdx.x & 31;
  const uint64_t warp = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const uint64_t nwarps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
  for (uint64_t s = warp; s < a.n_sent; s += nwarps) {
    const uint32_t w0 = a.sent_wbase[s], nw = a.sent_wcnt[s];
    uint32_t sum = 0;
    for (uint32_t i = lane; i < nw; i += 32) {
      const uint32_t w = w0 + i;
      sum += a.n_tok[rep ? rep[w] : w];
    }
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    if (lane == 0) a.n_ids[s] = (unsigned long long)sum + (a.bos ? 1 : 0) + (a.eos ? 1 : 0);
  }
}

__global__ void __launch_bounds__(256) emit_ids_kernel(EncArgs a, const uint32_t *__restrict__ rep,
                                                       const unsigned long long *__restrict__ out_off, int32_t *__restrict__ out) {
  const unsigned lane = threadIdx.x & 31;
  const uint64_t warp = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const uint64_t nwarps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
  for (uint64_t s = warp; s < a.n_sent; s += nwarps) {
    const uint32_t w0 = a.sent_wbase[s], nw = a.sent_wcnt[s];
    const unsigned long long ob = out_off[s], total = a.n_ids[s];
    auto at = [&](unsigned long long j) { return ob + (a.reverse ? total - 1 - j : j); };
    if (lane == 0) {
      if (a.bos) out[at(0)] = a.bos_id;
      if (a.eos) out[at(total - 1)] = a.eos_id;
    }
    unsigned long long pos = a.bos ? 1 : 0;
    for (uint32_t i0 = 0; i0 < nw; i0 += 32) {  // warp-uniform
      const uint32_t i = i0 + lane;
      uint32_t r = 0, n = 0;
      if (i < nw) {
        r = rep ? rep[w0 + i] : w0 + i;
        n = a.n_tok[r];
      }
      uint32_t x = n;
      for (int o = 1; o < 32; o <<= 1) {
        const uint32_t y = __shfl_up_sync(0xffffffffu, x, o);
        if ((int)lane >= o) x += y;
      }
      const uint32_t all = __shfl_sync(0xffffffffu, x, 31);
      if (n) {
        const int32_t *src = a.slots + ((uint64_t)a.word_pos[r] + 3ull * a.word_sent[r] + 1);
        const unsigned long long first = pos + (x - n);
        for (uint32_t k = 0; k < n; k++) out[at(first + k)] = src[k];
      }
      pos += all;
    }
  }
}

// yttm_enc_run: a chunk's id offsets are chunk-local; the ids in front of the chunk are added on the device before the
// offsets leave, so the host does no per-sentence work after the copies.
__global__ void __launch_bounds__(256) add_base_kernel(unsigned long long *__restrict__ off, uint64_t n, unsigned long long base) {
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) off[i] += base;
}

}  // namespace

namespace {

int enc_device(yttm_enc *enc, yttm_enc::Slot *e, const uint8_t *d_bytes, const uint64_t *d_offs, uint64_t n_bytes,
               uint64_t n_sent, int bos, int eos, int reverse, double dropout, uint64_t seed, uint64_t first_sentence,
               uint64_t *out_n) {
  yttm_ctx *c = enc->ctx;
  if (n_bytes >= 0xfffffff0ull || n_sent >= 0xfffffff0ull)
    YT_FAIL(c, "encode batch too large: at most 2^32 bytes / sentences per call (split the batch)");
  const uint64_t n_slots = n_bytes + 3 * n_sent;
  YT_CUDA(c, e->slots.reserve((n_slots + 8) * 4));
  YT_CUDA(c, e->ranks.reserve((n_slots + 8) * 4));
  if (dropout > 0) YT_CUDA(c, e->aux.reserve((n_slots + 8) * 24));
  const uint64_t max_words = n_bytes / 2 + n_sent + 8;
  YT_CUDA(c, e->wpos.reserve(max_words * 4));
  YT_CUDA(c, e->wsent.reserve(max_words * 4));
  YT_CUDA(c, e->nids.reserve((n_sent + 1) * 8));
  YT_CUDA(c, e->out_off.reserve((n_sent + 2) * 8));
  YT_CUDA(c, e->counter.reserve(64));
  YT_CUDA(c, cudaMemsetAsync(e->counter.p, 0, 64, c->stream));
  EncArgs a;
  a.bytes = d_bytes; a.offs = d_offs; a.n_sent = n_sent;
  a.slots = e->slots.as<int32_t>(); a.ranks = e->ranks.as<uint32_t>();
  a.aux = dropout > 0 ? e->aux.as<uint32_t>() : nullptr;
  a.word_pos = e->wpos.as<uint32_t>(); a.word_sent = e->wsent.as<uint32_t>();
  a.n_words = e->counter.as<unsigned long long>();
  a.n_ids = e->nids.as<unsigned long long>();
  a.cp2id = enc->cp2id.as<uint32_t>();
  a.rt.slots = enc->rules.as<uint4>(); a.rt.mask = enc->rule_mask;
  a.space_id = enc->space_id;
  a.unk_id = enc->unk; a.bos_id = enc->bos; a.eos_id = enc->eos;
  a.bos = bos; a.eos = eos; a.reverse = reverse;
  a.drop_thresh = dropout <= 0 ? 0 : (uint64_t)(dropout * 4294967296.0);
  a.seed = seed; a.first_sentence = first_sentence;
  *out_n = 0;
  auto *d_total = e->counter.as<unsigned long long>() + 1;
  if (n_sent == 0) return 0;
  ytc::timer_begin(c, "encode");
  YT_CUDA(c, e->swb.reserve((n_sent + 1) * 4));
  YT_CUDA(c, e->swc.reserve((n_sent + 1) * 4));
  a.sent_wbase = e->swb.as<uint32_t>();
  a.sent_wcnt = e->swc.as<uint32_t>();
  a.n_tok = nullptr;  // sized by the number of words, known after find_words_vec_kernel
  {
    ytc::timer_begin(c, "enc_find");
    const uint64_t blocks = std::min<uint64_t>((n_sent + 8 * FIND_SPW - 1) / (8 * FIND_SPW), (uint64_t)c->n_sm * 8);
    find_words_vec_kernel<<<(unsigned)std::max<uint64_t>(blocks, 1), 256, 0, c->stream>>>(a);
    ytc::timer_end(c, "enc_find");
    c->launches++;
  }
  unsigned long long n_words = 0;
  YT_CUDA(c, cudaMemcpyAsync(&n_words, a.n_words, 8, cudaMemcpyDeviceToHost, c->stream));
  YT_CUDA(c, cudaStreamSynchronize(c->stream));
  const uint32_t *d_rep = nullptr;  // dropout > 0: every word is its own representative
  if (n_words) {
    uint64_t blocks = std::min<uint64_t>((n_words + 127) / 128, (uint64_t)c->n_sm * 16);
    ytc::timer_begin(c, "enc_words");
    YT_CUDA(c, e->ntok.reserve(n_words * 4 + 16));
    a.n_tok = e->ntok.as<uint32_t>();
    if (a.drop_thresh == 0) {
      // words of more than LONG_W slots get a whole block each (a 16 KB word takes seconds on one thread)
      const uint32_t cap = (uint32_t)(n_bytes / LONG_W + 16);
      YT_CUDA(c, e->longw.reserve((size_t)cap * 16 + 16));
      LongList ll;
      ll.n = e->longw.as<unsigned long long>();
      ll.pos = reinterpret_cast<uint32_t *>(ll.n + 2);
      ll.sent = ll.pos + cap;
      ll.end = ll.sent + cap;
      ll.item = ll.end + cap;
      ll.cap = cap;
      YT_CUDA(c, cudaMemsetAsync(ll.n, 0, 8, c->stream));
      // table: 2 slots per occurrence up to 2^21 slots (16 MB, L2-resident); beyond that it works as a cache
      uint64_t tslots = std::max<uint64_t>(ytc::pow2ceil(std::min<uint64_t>(n_words, 1ull << 20) * 2), 1024);
      if (const char *env = std::getenv("YTTM_ENC_DEDUP_SLOTS")) tslots = ytc::pow2ceil((uint64_t)std::max(1, std::atoi(env)));  // tests: tiny tables
      YT_CUDA(c, e->dd_tab.reserve(tslots * 8));
      YT_CUDA(c, e->dd_rep.reserve(n_words * 4 + 16));
      YT_CUDA(c, e->dd_list.reserve(n_words * 4 + 16));
      DedupArgs d;
      d.tab = e->dd_tab.as<unsigned long long>(); d.mask = (uint32_t)(tslots - 1);
      d.rep = e->dd_rep.as<uint32_t>(); d.list = e->dd_list.as<uint32_t>();
      d.n_list = e->counter.as<unsigned long long>() + 2;  // zeroed with the other counters above
      d.weak_tag = std::getenv("YTTM_ENC_DEDUP_WEAKTAG") != nullptr;  // tests: tag collisions everywhere
      d_rep = d.rep;
      YT_CUDA(c, cudaMemsetAsync(d.tab, 0xff, tslots * 8, c->stream));
      ytc::timer_begin(c, "enc_dedup");
      dedup_words_kernel<<<(unsigned)blocks, 128, 0, c->stream>>>(a, n_words, d);
      ytc::timer_end(c, "enc_dedup");
      c->launches++;
      ytc::timer_begin(c, "enc_rep");
      encode_rep_words_kernel<<<(unsigned)blocks, 128, 0, c->stream>>>(a, d, ll);
      c->launches++;
      // no host round trip: the blocks read the list length themselves
      encode_long_words_kernel<<<(unsigned)c->n_sm, LONG_T, 0, c->stream>>>(a, ll);
      c->launches++;
      ytc::timer_end(c, "enc_rep");
    } else {
      encode_words_kernel<<<(unsigned)blocks, 128, 0, c->stream>>>(a, n_words);
      c->launches++;
    }
    ytc::timer_end(c, "enc_words");
  }
  const uint64_t sblocks = std::max<uint64_t>(std::min<uint64_t>((n_sent + 7) / 8, (uint64_t)c->n_sm * 8), 1);
  {  // per-sentence id counts from the words' token counts
    ytc::timer_begin(c, "enc_count");
    sentence_ids_kernel<<<(unsigned)sblocks, 256, 0, c->stream>>>(a, d_rep);
    ytc::timer_end(c, "enc_count");
    c->launches++;
  }
  // exclusive scan of the per-sentence id counts -> output offsets
  ytc::timer_begin(c, "enc_scan");
  if (yttm_device_scan_u64(c, a.n_ids, n_sent, e->out_off.as<unsigned long long>(), d_total)) return 1;
  ytc::timer_end(c, "enc_scan");
  unsigned long long total = 0;
  YT_CUDA(c, cudaMemcpyAsync(&total, d_total, 8, cudaMemcpyDeviceToHost, c->stream));
  YT_CUDA(c, cudaMemcpyAsync(e->out_off.as<unsigned long long>() + n_sent, d_total, 8, cudaMemcpyDeviceToDevice,
                             c->stream));
  YT_CUDA(c, cudaStreamSynchronize(c->stream));
  YT_CUDA(c, e->out_ids.reserve((total + 8) * 4));
  {
    ytc::timer_begin(c, "enc_gather");
    emit_ids_kernel<<<(unsigned)sblocks, 256, 0, c->stream>>>(a, d_rep, e->out_off.as<unsigned long long>(), e->out_ids.as<int32_t>());
    ytc::timer_end(c, "enc_gather");
    c->launches++;
  }
  ytc::timer_end(c, "encode");
  YT_CUDA(c, cudaGetLastError());
  *out_n = total;
  return 0;
}

}  // namespace

extern "C" {

int yttm_enc_create(yttm_ctx *c, const uint32_t *char_cp, const uint32_t *char_id, uint64_t n_chars,
                    const uint32_t *rules_xyz, uint64_t n_rules, int unk_id, int pad_id, int bos_id, int eos_id,
                    yttm_enc **out) {
  *out = nullptr;
  YT_CUDA(c, cudaSetDevice(c->device));
  yttm_enc *e = new yttm_enc();
  e->ctx = c;
  e->unk = unk_id; e->pad = pad_id; e->bos = bos_id; e->eos = eos_id;
  std::vector<uint32_t> tab(CP_LIMIT, NO_ID);
  bool have_space = false;
  for (uint64_t i = 0; i < n_chars; i++) {
    if (char_cp[i] >= CP_LIMIT) { delete e; YT_FAIL(c, "model: code point out of range"); }
    tab[char_cp[i]] = char_id[i];
    if (char_cp[i] == SPACE_CP) { e->space_id = char_id[i]; have_space = true; }
  }
  if (!have_space) { delete e; YT_FAIL(c, "model: U+2581 missing from char2id"); }
  e->h_char_cp.assign(char_cp, char_cp + n_chars);
  e->h_char_id.assign(char_id, char_id + n_chars);
  e->h_rules_xyz.assign(rules_xyz, rules_xyz + 3 * n_rules);
  e->vocab = n_chars + n_rules + (unk_id != -1) + (pad_id != -1) + (bos_id != -1) + (eos_id != -1);
  // 2 slots per rule of the open-addressed rule table (load <= 1/2, the measured configuration); most adjacent token
  // pairs have NO rule, and an unsuccessful linear-probe search costs ~2.5 probes at load 1/2, each probe a dependent
  // 16-byte load.
  const uint64_t per_rule = 2;
  uint64_t cap = std::max<uint64_t>(ytc::pow2ceil(n_rules * per_rule + 2), 1024);
  std::vector<uint4> slots(cap, make_uint4(0xffffffffu, 0xffffffffu, 0xffffffffu, 0));
  for (uint64_t i = 0; i < n_rules; i++) {
    uint32_t x = rules_xyz[3 * i], y = rules_xyz[3 * i + 1], z = rules_xyz[3 * i + 2];
    uint64_t h = rule_hash(x, y) & (cap - 1);
    bool dup = false;
    while (slots[h].x != 0xffffffffu) {
      if (slots[h].x == x && slots[h].y == y) { dup = true; break; }  // rule2id keeps the LAST index (bpe.cpp:1672)
      h = (h + 1) & (cap - 1);
    }
    if (dup) { slots[h].z = (uint32_t)i; slots[h].w = z; }
    else slots[h] = make_uint4(x, y, (uint32_t)i, z);
  }
  e->rule_mask = (uint32_t)(cap - 1);
  if (e->cp2id.reserve(CP_LIMIT * 4) != cudaSuccess || e->rules.reserve(cap * 16) != cudaSuccess) {
    delete e;
    YT_FAIL(c, "yttm_enc_create: out of device memory");
  }
  YT_CUDA(c, cudaMemcpyAsync(e->cp2id.p, tab.data(), CP_LIMIT * 4, cudaMemcpyHostToDevice, c->stream));
  YT_CUDA(c, cudaMemcpyAsync(e->rules.p, slots.data(), cap * 16, cudaMemcpyHostToDevice, c->stream));
  YT_CUDA(c, cudaStreamSynchronize(c->stream));
  *out = e;
  return 0;
}

void yttm_enc_destroy(yttm_enc *e) {
  if (!e) return;
  cudaSetDevice(e->ctx->device);
  e->cp2id.release();
  e->rules.release();
  yttm_dec_free(e->dec);
  for (int i = 0; i < 2; i++) {
    e->slot[i].release();
    if (e->ev_in[i]) cudaEventDestroy(e->ev_in[i]);
    if (e->ev_done[i]) cudaEventDestroy(e->ev_done[i]);
    if (e->ev_out[i]) cudaEventDestroy(e->ev_out[i]);
  }
  if (e->s_in) cudaStreamDestroy(e->s_in);
  if (e->s_out) cudaStreamDestroy(e->s_out);
  delete e;
}

int yttm_enc_run_device(yttm_enc *e, const char *d_bytes, const uint64_t *d_offsets, uint64_t n_bytes, uint64_t n_sent,
                        int bos, int eos, int reverse, double dropout, uint64_t seed, uint64_t first_sentence_index,
                        const int32_t **d_out_ids, const uint64_t **d_out_offsets, uint64_t *out_n) {
  if (!e) { g_yttm_create_error = "yttm_enc_run_device: null encoder handle (no CUDA device, or yttm_enc_create failed)"; return 1; }
  yttm_ctx *c = e->ctx;
  YT_CUDA(c, cudaSetDevice(c->device));
  if (bos && e->bos == -1) YT_FAIL(c, "Can't add <BOS> token. Model was trained without it.");
  if (eos && e->eos == -1) YT_FAIL(c, "Can't add <EOS> token. Model was trained without it.");
  if (enc_device(e, &e->slot[0], (const uint8_t *)d_bytes, d_offsets, n_bytes, n_sent, bos, eos, reverse, dropout,
                 seed, first_sentence_index, out_n))
    return 1;
  if (d_out_ids) *d_out_ids = e->slot[0].out_ids.as<int32_t>();
  if (d_out_offsets) *d_out_offsets = e->slot[0].out_off.as<uint64_t>();
  return 0;
}

int yttm_enc_run(yttm_enc *e, const char *bytes, const uint64_t *offsets, uint64_t n_sent, int bos, int eos, int reverse,
                 double dropout, uint64_t seed, uint64_t first_sentence_index, int32_t *out_ids, uint64_t out_cap,
                 uint64_t *out_offsets, uint64_t *out_n) {
  if (!e) { g_yttm_create_error = "yttm_enc_run: null encoder handle (no CUDA device, or yttm_enc_create failed)"; return 1; }
  yttm_ctx *c = e->ctx;
  YT_CUDA(c, cudaSetDevice(c->device));
  if (bos && e->bos == -1) YT_FAIL(c, "Can't add <BOS> token. Model was trained without it.");
  if (eos && e->eos == -1) YT_FAIL(c, "Can't add <EOS> token. Model was trained without it.");
  *out_n = 0;
  if (n_sent == 0) { if (out_offsets) out_offsets[0] = 0; return 0; }
  if (!e->s_in) {
    YT_CUDA(c, cudaStreamCreateWithFlags(&e->s_in, cudaStreamNonBlocking));
    YT_CUDA(c, cudaStreamCreateWithFlags(&e->s_out, cudaStreamNonBlocking));
    for (int i = 0; i < 2; i++) {
      YT_CUDA(c, cudaEventCreateWithFlags(&e->ev_in[i], cudaEventDisableTiming));
      YT_CUDA(c, cudaEventCreateWithFlags(&e->ev_done[i], cudaEventDisableTiming));
      YT_CUDA(c, cudaEventCreateWithFlags(&e->ev_out[i], cudaEventDisableTiming));
    }
  }
  // chunks of about CHUNK bytes, cut at sentence boundaries; chunk i lives in slot i & 1
  const uint64_t total_bytes = offsets[n_sent] - offsets[0];
  uint64_t chunk_bytes = 32ull << 20;
  if (const char *env = std::getenv("YTTM_ENC_CHUNK_MB")) chunk_bytes = (uint64_t)std::max(1, std::atoi(env)) << 20;
  std::vector<uint64_t> cut(1, 0);  // sentence indices
  while (cut.back() < n_sent) {
    const uint64_t lo = cut.back();
    const uint64_t want = offsets[lo] + chunk_bytes;
    uint64_t hi = (uint64_t)(std::upper_bound(offsets + lo + 1, offsets + n_sent + 1, want) - offsets) - 1;
    if (hi <= lo) hi = lo + 1;  // a single sentence longer than the chunk size
    if (offsets[n_sent] - offsets[hi] < chunk_bytes / 4) hi = n_sent;  // no tiny tail chunk
    cut.push_back(std::min<uint64_t>(hi, n_sent));
  }
  const size_t K = cut.size() - 1;
  c->timers["enc_chunks"].ms = (float)K;  // yttm_stage_ms(ctx, "enc_chunks"): how many chunks the last call used
  auto h2d = [&](size_t i) -> int {  // enqueue the input copies of chunk i on the copy-in stream
    yttm_enc::Slot &sl = e->slot[i & 1];
    const uint64_t lo = cut[i], hi = cut[i + 1], nb = offsets[hi] - offsets[lo];
    YT_CUDA(c, sl.d_bytes.reserve(nb + 64));
    YT_CUDA(c, sl.d_offs.reserve((hi - lo + 1) * 8));
    if (i >= 2) YT_CUDA(c, cudaStreamWaitEvent(e->s_in, e->ev_done[i & 1], 0));  // kernels of chunk i-2 are done with it
    if (nb) YT_CUDA(c, cudaMemcpyAsync(sl.d_bytes.p, bytes + offsets[lo], nb, cudaMemcpyHostToDevice, e->s_in));
    YT_CUDA(c, cudaMemcpyAsync(sl.d_offs.p, offsets + lo, (hi - lo + 1) * 8, cudaMemcpyHostToDevice, e->s_in));
    YT_CUDA(c, cudaEventRecord(e->ev_in[i & 1], e->s_in));
    return 0;
  };
  ytc::timer_begin(c, "e2e");
  if (h2d(0)) return 1;
  uint64_t base = 0;
  int rc_small = 0;
  for (size_t i = 0; i < K; i++) {
    yttm_enc::Slot &sl = e->slot[i & 1];
    const uint64_t lo = cut[i], hi = cut[i + 1], nb = offsets[hi] - offsets[lo];
    if (i + 1 < K && h2d(i + 1)) return 1;
    YT_CUDA(c, cudaStreamWaitEvent(c->stream, e->ev_in[i & 1], 0));
    if (i >= 2) YT_CUDA(c, cudaStreamWaitEvent(c->stream, e->ev_out[i & 1], 0));  // results of chunk i-2 have left
    uint64_t total = 0;
    if (enc_device(e, &sl, sl.d_bytes.as<uint8_t>(), sl.d_offs.as<uint64_t>(), nb, hi - lo, bos, eos, reverse, dropout,
                   seed, first_sentence_index + lo, &total))
      return 1;
    if (base && hi > lo) {  // chunk-local offsets -> batch offsets
      add_base_kernel<<<(unsigned)std::min<uint64_t>((hi - lo + 255) / 256, (uint64_t)c->n_sm * 4), 256, 0, c->stream>>>(
          sl.out_off.as<unsigned long long>(), hi - lo, (unsigned long long)base);
      c->launches++;
    }
    YT_CUDA(c, cudaEventRecord(e->ev_done[i & 1], c->stream));
    if (base + total > out_cap) rc_small = 2;
    if (!rc_small) {
      YT_CUDA(c, cudaStreamWaitEvent(e->s_out, e->ev_done[i & 1], 0));
      if (total)
        YT_CUDA(c, cudaMemcpyAsync(out_ids + base, sl.out_ids.p, total * 4, cudaMemcpyDeviceToHost, e->s_out));
      YT_CUDA(c, cudaMemcpyAsync(out_offsets + lo, sl.out_off.p, (hi - lo) * 8, cudaMemcpyDeviceToHost, e->s_out));
      YT_CUDA(c, cudaEventRecord(e->ev_out[i & 1], e->s_out));
    }
    base += total;
  }
  YT_CUDA(c, cudaStreamSynchronize(e->s_out));
  YT_CUDA(c, cudaStreamSynchronize(c->stream));
  ytc::timer_end(c, "e2e");
  *out_n = base;
  if (rc_small) { c->err = "yttm_enc_run: output buffer too small"; return 2; }
  out_offsets[n_sent] = base;
  (void)total_bytes;
  return 0;
}

}  // extern "C"
