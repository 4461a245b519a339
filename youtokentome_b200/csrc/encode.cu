// encode.cu — hot path (b): batch encode_as_ids on one H100.
//
// Replaces BaseEncoder::encode_parallel / encode_sentence (youtokentome/cpp/bpe.cpp:1697-1738,
// 1455-1632) behind yttm_enc_run* of include/yttm_b200.h.  The reference gives each CPU thread a
// contiguous range of sentences and runs a heap-driven merge loop per word.  Here the batch is
// one flat byte buffer in HBM and the unit of parallel work is the WORD:
//   find_words_vec_kernel       block per group of sentences staged in shared memory: word starts (on raw bytes, see
//                               bpe_core.cuh) go to a global work list in byte order, one reservation per group;
//                               every sentence records its range of work items
//   dropout = 0 (the ids of a word are a function of its bytes, so every distinct word is encoded once):
//     dedup_words_kernel        elects one representative occurrence per distinct word (16-byte vector loads)
//     encode_rep_words_kernel   one thread per representative: UTF-8 decode -> char ids (unknown runs collapse to
//                               one pseudo token, bpe.cpp:1513-1533) -> min-rank merge loop, leftmost first
//                               (MergeEvent2::operator< bpe.cpp:1475-1478)
//     encode_long_words_kernel  one block per representative of more than LONG_W slots
//   dropout > 0 (every occurrence draws for itself):
//     encode_words_kernel       one thread per occurrence, the same merge loop with BPE-dropout (DropoutQueue
//                               bpe.cpp:1417-1453 with a counter-based generator)
//   every encoded item leaves a 16-byte record (id count, first three ids), so most words are served by one load
//   emit_ids_kernel             single pass, block per tile of 256 sentences: id counts from the records, the tile's
//                               output offset by a decoupled look-back over the earlier tiles, then offsets and ids
// yttm_enc_run_padded* replace it with
//   emit_padded_kernel          block per tile of 256 sentences, row i of an [n_sent, L] matrix at i L: the tiles need
//                               nothing from each other (no look-back); a counting form finds L when it is not given
// On request (yttm_enc_run_spans* / yttm_enc_run_subwords*) the same flow also gives the source span of every id and
// the subword pieces:
//   span_words_kernel           one thread per encoded word: the span of each of its ids relative to the word start
//   emit_ids_kernel<true>       ... and the spans at the occurrences' positions
//   sub_count_kernel / scan / sub_emit_kernel   one thread per id: piece lengths, offsets, piece bytes
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
  uint32_t *sent_wbase;       // first work item / number of work items of every sentence
  uint32_t *sent_wcnt;
  uint4 *rec;                 // per encoded work item (every representative, or every word with dropout): (number of
                              // ids, first three ids), so that a word of at most 3 ids is one 16-byte load (put_rec)
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

// the record of an encoded item from its n final ids t[0 ..] (ids past n read as 0)
__device__ __forceinline__ void put_rec(uint4 *rec, uint64_t w, uint32_t n, const int32_t *t) {
  rec[w] = make_uint4(n, n > 0 ? (uint32_t)t[0] : 0u, n > 1 ? (uint32_t)t[1] : 0u, n > 2 ? (uint32_t)t[2] : 0u);
}

// exclusive sum of one value per thread over the block; *tot = block sum (starts with a barrier, so s_red may be reused
// right after the previous call)
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

// Word starts: one block per GROUP of G consecutive sentences (G from the batch's mean sentence length, so that a
// typical group fits one FIND_TILE-byte piece).  The block stages the group's bytes in shared memory with aligned
// 16-byte loads (every byte is read from HBM once), each thread decides the word starts of FIND_BPT consecutive staged
// bytes, one block-wide scan numbers them in byte order and ONE atomicAdd per group reserves the group's range of the
// work list, so the words of every sentence are a contiguous run of work items.  A group longer than a piece (long
// sentences) is streamed piece by piece twice: count, reserve, write.  word_start_at(p) == space_before(p) &&
// !space_at(p) on raw bytes (a continuation byte is never a space); the sentence bounds inside a group come from a
// shared bitmap of sentence starts: a sentence start is always preceded by a space, and an E2 96 81 across a sentence
// start is a space unit on neither side.  The group's first byte and its end are sentence starts of the bitmap, so the
// bytes outside the group decide nothing and no halo from neighbouring groups is needed.
constexpr int FIND_T = 256;                   // threads per block
constexpr int FIND_BPT = 64;                  // bytes per thread and piece (one 64-bit mask)
constexpr int FIND_TILE = FIND_T * FIND_BPT;  // bytes per piece (16 KB)
constexpr int FIND_HALO = 16;                 // staged bytes on either side of a piece (the rules look 3 back, 2 ahead)
constexpr int FIND_BUF = FIND_TILE + 2 * FIND_HALO;
constexpr uint32_t FIND_GMAX = 256;           // sentences per group at most
static_assert(FIND_BPT == 64 && FIND_HALO % 32 == 16, "a thread's 64 bitmap bits start at bit 16 of a bitmap word");
// set bits / lowest set bit (m != 0) of a thread's 64-bit mask, from the 32-bit intrinsics
__device__ __forceinline__ uint32_t find_popc64(uint64_t m) { return __popc((uint32_t)m) + __popc((uint32_t)(m >> 32)); }
__device__ __forceinline__ int find_low64(uint64_t m) {
  return (uint32_t)m ? __ffs((int)(uint32_t)m) - 1 : 31 + __ffs((int)(uint32_t)(m >> 32));
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
// staged byte i: is it a space unit / does a space unit end right before it (sentence starts from the bitmap sb)
__device__ __forceinline__ bool find_sbit(const uint32_t *sb, int i) { return (sb[i >> 5] >> (i & 31)) & 1u; }
__device__ __forceinline__ bool find_at(const uint8_t *b, const uint32_t *sb, int i) {
  return is_space_byte(b[i]) ||
         (b[i] == 0xe2 && b[i + 1] == 0x96 && b[i + 2] == 0x81 && !find_sbit(sb, i + 1) && !find_sbit(sb, i + 2));
}
__device__ __forceinline__ bool find_before(const uint8_t *b, const uint32_t *sb, int i) {
  return find_sbit(sb, i) || is_space_byte(b[i - 1]) ||
         (b[i - 3] == 0xe2 && b[i - 2] == 0x96 && b[i - 1] == 0x81 && !find_sbit(sb, i - 2) && !find_sbit(sb, i - 1));
}

// Stages the piece [pa, pa + FIND_TILE) of the group [gstart, gend), FIND_HALO bytes on either side (the address of
// batch byte pa is 16-byte aligned), and the bitmap of the sentence starts among them; returns the word starts among
// the thread's FIND_BPT bytes (bit j = batch byte pa + FIND_BPT * threadIdx.x + j).  Starts with a barrier: the
// previous piece is done with the buffers.
__device__ __forceinline__ uint64_t find_piece(const uint8_t *bytes, int64_t n_total, int64_t pa, int64_t gstart,
                                               int64_t gend, const uint32_t *s_off, uint32_t ng, uint4 *s_buf,
                                               uint32_t *s_sb) {
  constexpr int NCH = FIND_BUF / 16, PER = (NCH + FIND_T - 1) / FIND_T;
  const int64_t p0 = pa - FIND_HALO;  // batch position of staged byte 0
  const int tid = (int)threadIdx.x;
  __syncthreads();
  uint4 v[PER];
#pragma unroll
  for (int r = 0; r < PER; r++) {  // every load first: PER 16-byte loads in flight per thread
    const int j = tid + r * FIND_T;
    const int64_t q = p0 + 16 * (int64_t)j;
    v[r] = make_uint4(0u, 0u, 0u, 0u);
    if (j < NCH && q + 16 > gstart && q < gend) {  // only chunks holding bytes of the group
      if (q >= 0 && q + 16 <= n_total) {
        v[r] = *reinterpret_cast<const uint4 *>(bytes + q);
      } else {  // a chunk over an end of the batch: byte by byte, never outside it
        uint32_t w0 = 0, w1 = 0, w2 = 0, w3 = 0;
#pragma unroll
        for (int k = 0; k < 16; k++)
          if (q + k >= 0 && q + k < n_total) {
            const uint32_t b = (uint32_t)bytes[q + k] << (8 * (k & 3));
            if (k < 4) w0 |= b; else if (k < 8) w1 |= b; else if (k < 12) w2 |= b; else w3 |= b;
          }
        v[r] = make_uint4(w0, w1, w2, w3);
      }
    }
  }
#pragma unroll
  for (int r = 0; r < PER; r++)
    if (tid + r * FIND_T < NCH) s_buf[tid + r * FIND_T] = v[r];
  for (int j = tid; j < FIND_BUF / 32 + 1; j += FIND_T) s_sb[j] = 0u;
  __syncthreads();
  for (uint32_t i = (uint32_t)tid; i <= ng; i += FIND_T) {
    const int64_t x = (int64_t)s_off[i] - p0;
    if (x >= 0 && x < FIND_BUF) atomicOr(s_sb + (x >> 5), 1u << (x & 31));
  }
  __syncthreads();
  const int64_t lo = pa + FIND_BPT * (int64_t)tid;  // batch position of the thread's first byte
  const int64_t b = gstart - lo, e = gend - lo;    // the group's bytes among the thread's: [bb, ee)
  const int bb = b < 0 ? 0 : b > FIND_BPT ? FIND_BPT : (int)b, ee = e < 0 ? 0 : e > FIND_BPT ? FIND_BPT : (int)e;
  if (ee <= bb) return 0;
  const uint64_t inside = (ee - bb == 64 ? ~0ull : (1ull << (ee - bb)) - 1) << bb;
  const int i0 = FIND_HALO + FIND_BPT * tid;  // staged index of the thread's first byte
  const uint32_t prev = reinterpret_cast<const uint32_t *>(s_buf)[i0 / 4 - 1];
  uint32_t e2 = swar_eq(prev, 0xe2e2e2e2u);
  uint64_t sp = 0;
#pragma unroll
  for (int k = 0; k < FIND_BPT / 16; k++) {
    const uint4 c = s_buf[i0 / 16 + k];
    e2 |= swar_eq(c.x, 0xe2e2e2e2u) | swar_eq(c.y, 0xe2e2e2e2u) | swar_eq(c.z, 0xe2e2e2e2u) | swar_eq(c.w, 0xe2e2e2e2u);
    sp |= (uint64_t)(swar_mask4(swar_space(c.x)) | swar_mask4(swar_space(c.y)) << 4 | swar_mask4(swar_space(c.z)) << 8 |
                     swar_mask4(swar_space(c.w)) << 12) << (16 * k);
  }
  if (!(e2 & 0x80808080u)) {
    // no 0xE2 from four bytes before on, so no U+2581 touches these bytes: a word starts where a sentence starts or an
    // ASCII space is followed by a non-space byte
    const uint32_t *sw = s_sb + (i0 >> 5);
    const uint64_t starts = (uint64_t)(sw[0] >> 16) | ((uint64_t)sw[1] << 16) | ((uint64_t)sw[2] << 48);
    return (starts | (sp << 1) | (swar_space(prev) >> 31)) & ~sp & inside;
  }
  const uint8_t *sbyte = reinterpret_cast<const uint8_t *>(s_buf);
  uint64_t f = 0;
  for (int j = bb; j < ee; j++)
    if (find_before(sbyte, s_sb, i0 + j) && !find_at(sbyte, s_sb, i0 + j)) f |= 1ull << j;
  return f;
}

// (4 blocks of 256 threads per SM, the occupancy it is built for: 2 x 16 KB of staged bytes per SM in flight)
__global__ void __launch_bounds__(FIND_T, 4) find_words_vec_kernel(EncArgs a, uint32_t G) {
  __shared__ uint4 s_buf[FIND_BUF / 16];
  __shared__ uint32_t s_sb[FIND_BUF / 32 + 1];
  __shared__ uint32_t s_off[FIND_GMAX + 1];  // the group's sentence starts (batch positions), s_off[ng] = its end
  __shared__ uint32_t s_wb[FIND_GMAX + 1];   // words of the group in front of them
  __shared__ uint32_t s_red[FIND_T / 32];
  __shared__ unsigned long long s_base;
  constexpr int64_t FAR = (int64_t)1 << 62;
  const int tid = (int)threadIdx.x;
  const uint64_t o0 = a.offs[0];
  const int64_t n_total = (int64_t)(a.offs[a.n_sent] - o0);
  const int64_t mis = (int64_t)(reinterpret_cast<uintptr_t>(a.bytes) & 15u);
  for (uint64_t g = (uint64_t)blockIdx.x * G; g < a.n_sent; g += (uint64_t)gridDim.x * G) {  // block-uniform
    const uint32_t ng = (uint32_t)min((uint64_t)G, a.n_sent - g);
    __syncthreads();  // the previous group is done with s_off / s_wb / s_base
    for (uint32_t i = (uint32_t)tid; i <= ng; i += FIND_T) s_off[i] = (uint32_t)(a.offs[g + i] - o0);
    __syncthreads();
    const int64_t gstart = s_off[0], gend = s_off[ng];
    const int64_t a0 = gstart - ((gstart + mis) & 15);  // the address of batch byte a0 is 16-byte aligned
    const uint32_t np = gend - a0 > FIND_TILE ? (uint32_t)((gend - a0 + FIND_TILE - 1) / FIND_TILE) : 1u;
    uint32_t tot;
    if (np > 1) {  // a group longer than a piece: count, then reserve before the write pass
      uint32_t total = 0;
      for (uint32_t k = 0; k < np; k++) {
        const uint64_t m = find_piece(a.bytes, n_total, a0 + (int64_t)k * FIND_TILE, gstart, gend, s_off, ng, s_buf, s_sb);
        long_block_scan_sum(find_popc64(m), s_red, &tot);
        total += tot;
      }
      if (tid == 0) s_base = total ? atomicAdd(a.n_words, (unsigned long long)total) : 0ull;
    }
    uint32_t run = 0;  // words of the group in the earlier pieces
    for (uint32_t k = 0; k < np; k++) {
      const int64_t pa = a0 + (int64_t)k * FIND_TILE;
      uint64_t m = find_piece(a.bytes, n_total, pa, gstart, gend, s_off, ng, s_buf, s_sb);
      uint32_t n = run + long_block_scan_sum(find_popc64(m), s_red, &tot);  // words of the group before mine
      if (np == 1) {
        if (tid == 0) s_base = tot ? atomicAdd(a.n_words, (unsigned long long)tot) : 0ull;
        __syncthreads();
      }
      const unsigned long long base = s_base;
      // the thread's bytes in order: a sentence start among them records the words in front of it, a word belongs to
      // the sentence of the last start at or before it (the last thread of the last piece also takes the group's end)
      const int64_t lo = pa + FIND_BPT * (int64_t)tid;
      const int64_t lim = k + 1 == np && tid == FIND_T - 1 ? FAR : lo + FIND_BPT;
      uint32_t i = 0, r = ng + 1;  // i = first sentence start at or after lo
      while (i < r) {
        const uint32_t mid = (i + r) >> 1;
        if ((int64_t)s_off[mid] < lo) i = mid + 1; else r = mid;
      }
      while (true) {
        const int64_t x = i <= ng ? (int64_t)s_off[i] : FAR;
        const int64_t p = m ? lo + find_low64(m) : FAR;
        if (x < lim && x <= p) { s_wb[i++] = n; continue; }
        if (!m) break;
        a.word_pos[base + n] = (uint32_t)p;
        a.word_sent[base + n] = (uint32_t)(g + i - 1);
        n++;
        m &= m - 1;
      }
      run += tot;
    }
    __syncthreads();
    const unsigned long long base = s_base;
    for (uint32_t i = (uint32_t)tid; i < ng; i += FIND_T) {
      a.sent_wbase[g + i] = (uint32_t)(base + s_wb[i]);
      a.sent_wcnt[g + i] = s_wb[i + 1] - s_wb[i];
    }
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
    put_rec(a.rec, w, n, t);
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
// inclusive max of one value per thread over the block (long_block_scan_sum, above, is the exclusive sum)
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
    __syncthreads();  // t[0 .. 2] are final
    if (threadIdx.x == 0) put_rec(a.rec, ll.item[w], n_out, reinterpret_cast<const int32_t *>(t));
    __syncthreads();
  }
}

// Dropout = 0: every distinct word of the batch is encoded ONCE.  Without dropout the ids of a word are a pure function
// of its bytes [p0, q): a lead byte whose announced length reaches past q sees either the end of the sentence or the
// first byte of a space unit (never a continuation byte), INVALID_CP with length 1 in both cases (decode_unit), so
// nothing outside the word enters.  Natural text repeats its words (the bench batch: 20 M occurrences of < 200 k
// words), and the merge loop of encode_word is the expensive part of encoding a word.  Three launches:
//   dedup_words_kernel       one thread per occurrence: end of the word + 64-bit hash of its bytes; an
//                            open-addressed table of (32-bit tag, work item) words, small enough to stay in L2, elects
//                            the first occurrence that claims a slot as the word's representative; later occurrences
//                            with the same tag compare BYTES with it (exactness never rests on the hash).  A word that
//                            finds neither itself nor a free slot within DEDUP_PROBES probes represents itself, so the
//                            table is a bounded cache, not a limit.
//   encode_rep_words_kernel  the per-word body, over the representatives only (list length read on the device);
//                            representatives of more than LONG_W slots go to the list of encode_long_words_kernel
//   encode_long_words_kernel a block per long representative
// emit_ids_kernel then copies the ids of a representative (its record, or its slots) to every occurrence.  The slot of the first token of work
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

// The words' bytes are read 16 at a time: aligned 16-byte loads (lanes whose words are neighbours share their lines)
// and a shift that lines the bytes up, never a byte-serial gather.
struct Chunk16 { uint64_t lo, hi; };  // 16 bytes, little-endian
// the 16 bytes from batch position q (the address of byte q is 16-byte aligned); bytes outside the batch read as 0
__device__ __forceinline__ Chunk16 dd_chunk(const uint8_t *s, int64_t q, int64_t n_total) {
  if (q >= 0 && q + 16 <= n_total) {
    const uint4 v = *reinterpret_cast<const uint4 *>(s + q);
    return Chunk16{v.x | (uint64_t)v.y << 32, v.z | (uint64_t)v.w << 32};
  }
  Chunk16 c{0, 0};  // a chunk over an end of the batch: byte by byte, never outside it
#pragma unroll
  for (int k = 0; k < 16; k++)
    if (q + k >= 0 && q + k < n_total) {
      if (k < 8) c.lo |= (uint64_t)s[q + k] << (8 * k);
      else c.hi |= (uint64_t)s[q + k] << (8 * (k - 8));
    }
  return c;
}
// bytes o .. o + n - 1 of the 32 bytes c0:c1 (o < 16, 1 <= n <= 16), zero above
__device__ __forceinline__ Chunk16 dd_shift(Chunk16 c0, Chunk16 c1, uint32_t o, uint32_t n) {
  const uint64_t x0 = o >= 8 ? c0.hi : c0.lo, x1 = o >= 8 ? c1.lo : c0.hi, x2 = o >= 8 ? c1.hi : c1.lo;
  const uint32_t s = 8 * (o & 7);
  Chunk16 r = s ? Chunk16{(x0 >> s) | (x1 << (64 - s)), (x1 >> s) | (x2 << (64 - s))} : Chunk16{x0, x1};
  if (n <= 8) { r.hi = 0; if (n < 8) r.lo &= (1ull << (8 * n)) - 1; }
  else if (n < 16) r.hi &= (1ull << (8 * (n - 8))) - 1;
  return r;
}
// the n (1 .. 16) bytes at batch position p; mis = address of the batch & 15
__device__ __forceinline__ Chunk16 dd_window(const uint8_t *s, int64_t p, uint32_t n, int64_t n_total, int64_t mis) {
  const uint32_t o = (uint32_t)((p + mis) & 15);
  const Chunk16 c0 = dd_chunk(s, p - o, n_total);
  const Chunk16 c1 = o + n > 16 ? dd_chunk(s, p - o + 16, n_total) : Chunk16{0, 0};
  return dd_shift(c0, c1, o, n);
}
// 16-bit masks of the bytes of a chunk that are ASCII spaces / equal a given byte (v4 = the byte four times)
__device__ __forceinline__ uint32_t dd_space16(Chunk16 c) {
  return swar_mask4(swar_space((uint32_t)c.lo)) | swar_mask4(swar_space((uint32_t)(c.lo >> 32))) << 4 |
         swar_mask4(swar_space((uint32_t)c.hi)) << 8 | swar_mask4(swar_space((uint32_t)(c.hi >> 32))) << 12;
}
__device__ __forceinline__ uint32_t dd_eq16(Chunk16 c, uint32_t v4) {
  return swar_mask4(swar_eq((uint32_t)c.lo, v4)) | swar_mask4(swar_eq((uint32_t)(c.lo >> 32), v4)) << 4 |
         swar_mask4(swar_eq((uint32_t)c.hi, v4)) << 8 | swar_mask4(swar_eq((uint32_t)(c.hi >> 32), v4)) << 12;
}
__device__ __forceinline__ uint64_t dd_rotl(uint64_t x, int r) { return (x << r) | (x >> (64 - r)); }

__global__ void __launch_bounds__(128) dedup_words_kernel(EncArgs a, uint64_t n_words, DedupArgs d) {
  const unsigned lane = threadIdx.x & 31;
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  const uint64_t o0 = a.offs[0];
  const int64_t n_total = (int64_t)(a.offs[a.n_sent] - o0);
  const int64_t mis = (int64_t)(reinterpret_cast<uintptr_t>(a.bytes) & 15u);
  for (uint64_t w0 = (uint64_t)blockIdx.x * blockDim.x + (threadIdx.x & ~31u); w0 < n_words; w0 += stride) {  // warp-uniform
    const uint64_t w = w0 + lane;
    bool is_rep = false;
    if (w < n_words) {
      const int64_t p0 = a.word_pos[w], hi = (int64_t)(a.offs[(uint64_t)a.word_sent[w] + 1] - o0);
      uint32_t l;
      // ---- end of the word: the first space unit at or after p0, or hi; its first 3 chunks stay in registers
      const uint32_t o = (uint32_t)((p0 + mis) & 15);
      Chunk16 c0{0, 0}, c1{0, 0}, c2{0, 0};
      int64_t end = hi;
      for (int64_t q = p0 - o, k = 0; q < hi; q += 16, k++) {
        const Chunk16 c = dd_chunk(a.bytes, q, n_total);
        if (k == 0) c0 = c; else if (k == 1) c1 = c; else if (k == 2) c2 = c;
        const int64_t lim = hi - q;  // bytes of the sentence in this chunk (if below 16)
        uint32_t m = dd_space16(c);
        const uint32_t e2 = dd_eq16(c, 0xe2e2e2e2u);
        if (e2) {  // U+2581 = E2 96 81 inside the sentence; one starting in the last two bytes is checked byte by byte
          const uint32_t whole = lim - 2 >= 14 ? 0x3fffu : lim - 2 <= 0 ? 0u : (1u << (lim - 2)) - 1;
          m |= e2 & (dd_eq16(c, 0x96969696u) >> 1) & (dd_eq16(c, 0x81818181u) >> 2) & whole;
          for (int j = 14; j < 16; j++)
            if (((e2 >> j) & 1u) && j < lim && space_at(a.bytes, (uint64_t)(q + j), (uint64_t)hi, &l)) m |= 1u << j;
        }
        if (k == 0) m &= 0xffffu << o;
        if (lim < 16) m &= (1u << lim) - 1;
        if (m) { end = q + __ffs((int)m) - 1; break; }
      }
      const uint32_t len = (uint32_t)(end - p0);
      // bytes 16 k .. of the word (n of them)
      auto own = [&](uint32_t k, uint32_t n) {
        return k == 0 ? dd_shift(c0, c1, o, n) : k == 1 ? dd_shift(c1, c2, o, n)
                                                        : dd_window(a.bytes, p0 + 16 * (int64_t)k, n, n_total, mis);
      };
      uint64_t h = len * 0x9e3779b97f4a7c15ull;  // a function of the word's bytes only
      for (uint32_t k = 0; 16ull * k < len; k++) {
        const Chunk16 x = own(k, min(16u, len - 16 * k));
        h = (dd_rotl(h, 23) ^ x.lo) * 0x9e3779b97f4a7c15ull;
        h = (dd_rotl(h, 23) ^ x.hi) * 0xc2b2ae3d27d4eb4full;
      }
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
        bool same = p2 + len <= hi2;
        for (uint32_t k = 0; same && 16ull * k < len; k++) {
          const uint32_t n = min(16u, len - 16 * k);
          const Chunk16 x = dd_window(a.bytes, (int64_t)p2 + 16 * (int64_t)k, n, n_total, mis), y = own(k, n);
          same = x.lo == y.lo && x.hi == y.hi;
        }
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
    if (owned > LONG_W) {  // a whole block will take it (encode_long_words_kernel writes its record)
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
    put_rec(a.rec, w, n, t);
  }
}

// ---- spans ------------------------------------------------------------------------------------------------------
// The source bytes of every id: span_words_kernel walks the units of every encoded item (a representative, or every
// occurrence with dropout) in step with its ids and writes each id's span relative to the word start into the slot
// beside the id (rel, same indexing as slots).  The span of a word's ids is a function of the word's bytes and ids, so
// the occurrences of a representative share it; emit_ids_kernel<true> adds the occurrence's position.
//   ordinary id  covers units[id] valid units (its recipe without the word-initial U+2581); an invalid unit between
//                two of them lies inside its span, one in front of its first unit lies in no span
//   unk id       covers the maximal run of out-of-alphabet valid units that starts at the next valid unit
//   units = 0    the word-initial "▁" no rule merged: the empty span at the next valid unit
struct alignas(16) Span64 { unsigned long long lo, hi; };  // (start, end), one 16-byte store
struct SpanOut {
  uint2 *rel;                    // per slot: (start, end) relative to the word start
  const uint32_t *units;         // per id
  Span64 *spans;                 // per output id: (start, end) in the coordinates of offs
};

__global__ void __launch_bounds__(128) span_words_kernel(EncArgs a, const uint32_t *__restrict__ list,
                                                         const unsigned long long *__restrict__ n_list, uint64_t n_items,
                                                         SpanOut so) {
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  const uint64_t o0 = a.offs[0];
  const uint64_t n = list ? *n_list : n_items;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const uint32_t w = list ? list[i] : (uint32_t)i;
    const uint64_t p0 = a.word_pos[w], s = a.word_sent[w];
    const uint64_t hi = a.offs[s + 1] - o0;
    const uint64_t slot0 = p0 + 3 * s + 1;
    const int32_t *t = a.slots + slot0;
    uint2 *rel = so.rel + slot0;
    const uint32_t n_tok = a.rec[w].x;
    // the first valid unit at or after q inside the word: its start (hi if none), code point and length
    auto next_valid = [&](uint64_t q, uint32_t *cp, uint32_t *l) {
      while (q < hi && !space_at(a.bytes, q, hi, l)) {
        *cp = decode_unit(a.bytes, q, hi, l);
        if (*cp != INVALID_CP) return q;
        q += *l;
      }
      return hi;
    };
    uint64_t q = p0;
    for (uint32_t k = 0; k < n_tok; k++) {
      const int32_t id = t[k];
      uint32_t cp = 0, l = 0;
      uint64_t u = next_valid(q, &cp, &l);
      const uint64_t start = u;
      uint64_t end = u;
      if (id == a.unk_id) {
        while (u < hi && a.cp2id[cp] == NO_ID) { end = u + l; u = next_valid(end, &cp, &l); }
      } else {
        for (uint32_t m = so.units[id]; m && u < hi; m--) { end = u + l; if (m > 1) u = next_valid(end, &cp, &l); }
      }
      q = end;
      rel[k] = make_uint2((uint32_t)(start - p0), (uint32_t)(end - p0));
    }
  }
}

// ---- output ---------------------------------------------------------------------------------------------------
// The words of sentence s are the work items [sent_wbase[s], + sent_wcnt[s]) in byte order (find_words_vec_kernel); the
// ids of work item w are those of its representative r = rep[w] (r = w with dropout): rec[r].x of them, the first three
// in rec[r] itself, all of them at slot(word_pos[r] + 3 word_sent[r] + 1).  One single-pass kernel takes them from the
// encoded words straight to the packed output, without compacting the slot buffer and without a host round trip:
//   emit_ids_kernel   a block per tile of EMIT_T consecutive sentences, taken in ticket order: the ids of the tile's
//                     sentences (a thread per word), a decoupled look-back over the earlier tiles for the tile's output
//                     offset, then out_off and the ids (and the spans), a thread per word again.  The last tile writes
//                     out_off[n_sent] and the batch's total.
// Tiles publish one 64-bit word each: flag bits over a 62-bit id count, so value and flag are never seen apart and
// no fence is needed.  Only the order of the look-back words matters: nothing else a block writes is read in the launch.
constexpr int EMIT_T = 256;                                  // threads per block = sentences per tile
constexpr unsigned long long LB_AGG = 1ull << 62;            // the tile's own id count
constexpr unsigned long long LB_PRE = 1ull << 63;            // ids of the tiles up to and including this one
constexpr unsigned long long LB_VAL = LB_AGG - 1;            // (0 = not published yet)
struct EmitArgs {
  const uint32_t *rep;         // null with dropout (every word represents itself)
  unsigned long long *tiles;   // look-back word per tile, zeroed before the launch
  unsigned long long *ticket;  // zeroed before the launch
  unsigned long long *total;   // ids of the batch (the last tile)
  unsigned long long *out_off; // n_sent + 1
  int32_t *out;
};

// exclusive sum over the block of EMIT_T threads; *tot = block sum (starts with a barrier, like long_block_scan_sum)
__device__ __forceinline__ unsigned long long emit_block_scan(unsigned long long v, unsigned long long *s_red,
                                                              unsigned long long *tot) {
  const unsigned lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  unsigned long long x = v;
  for (int o = 1; o < 32; o <<= 1) { const unsigned long long y = __shfl_up_sync(0xffffffffu, x, o); if ((int)lane >= o) x += y; }
  __syncthreads();
  if (lane == 31) s_red[wid] = x;
  __syncthreads();
  unsigned long long base = 0, all = 0;
  for (unsigned i = 0; i < EMIT_T / 32; i++) { const unsigned long long w = s_red[i]; if (i < wid) base += w; all += w; }
  *tot = all;
  return base + x - v;
}

template <bool SPANS>
__global__ void __launch_bounds__(EMIT_T) emit_ids_kernel(EncArgs a, EmitArgs e, SpanOut so) {
  __shared__ uint32_t s_wb[EMIT_T];             // first work item of each sentence of the tile
  __shared__ uint32_t s_wofs[EMIT_T + 1];       // words of the tile in front of each sentence
  __shared__ uint32_t s_ids[EMIT_T];            // ids of each sentence's words
  __shared__ unsigned long long s_off[EMIT_T];  // ids of the tile in front of each sentence
  __shared__ unsigned long long s_red[EMIT_T / 32];
  __shared__ unsigned long long s_tile, s_base;
  const uint32_t tid = threadIdx.x;
  if (tid == 0) s_tile = atomicAdd(e.ticket, 1ull);  // blocks do not start in blockIdx order
  s_ids[tid] = 0;
  __syncthreads();
  const uint64_t tile = s_tile, s0 = tile * EMIT_T;
  const uint32_t ns = (uint32_t)min((uint64_t)EMIT_T, a.n_sent - s0);
  const uint32_t be = (a.bos ? 1u : 0u) + (a.eos ? 1u : 0u);
  const uint32_t *rep = e.rep;
  uint32_t wc = 0;
  if (tid < ns) { s_wb[tid] = a.sent_wbase[s0 + tid]; wc = a.sent_wcnt[s0 + tid]; }
  unsigned long long tw;
  const uint32_t wofs = (uint32_t)emit_block_scan(wc, s_red, &tw);
  const uint32_t n_tw = (uint32_t)tw;  // words of the tile
  if (tid < ns) s_wofs[tid] = wofs;
  if (tid == 0) s_wofs[ns] = n_tw;
  __syncthreads();
  // the tile's j-th word: its sentence k (the last one with s_wofs[k] <= j: empty sentences in front of it share its
  // s_wofs) and its work item
  auto word = [&](uint32_t j, uint32_t *k) {
    uint32_t lo = 0, hi = ns;
    while (hi - lo > 1) { const uint32_t mid = (lo + hi) >> 1; if (s_wofs[mid] <= j) lo = mid; else hi = mid; }
    *k = lo;
    return s_wb[lo] + (j - s_wofs[lo]);
  };
  for (uint32_t j = tid; j < n_tw; j += EMIT_T) {
    uint32_t k;
    const uint32_t w = word(j, &k);
    atomicAdd(&s_ids[k], a.rec[rep ? rep[w] : w].x);
  }
  __syncthreads();
  const uint32_t cnt = tid < ns ? s_ids[tid] + be : 0u;  // ids of my sentence
  unsigned long long agg;
  const unsigned long long off = emit_block_scan(cnt, s_red, &agg);
  // ---- decoupled look-back (warp 0): the ids of the tiles in front of this one
  if (tid < 32) {
    unsigned long long excl = 0;
    if (tile > 0) {
      if (tid == 0) *(volatile unsigned long long *)(e.tiles + tile) = LB_AGG | agg;
      for (int64_t look = (int64_t)tile - 1;; look -= 32) {
        const int64_t i = look - (int64_t)tid;
        unsigned long long v;
        do {  // the 32 tiles in front, nearest first (before tile 0: an inclusive prefix of 0)
          v = LB_PRE;
          if (i >= 0) v = *(volatile unsigned long long *)(e.tiles + i);
        } while (__ballot_sync(0xffffffffu, v == 0));
        const unsigned pm = __ballot_sync(0xffffffffu, (v & LB_PRE) != 0);
        const unsigned take = pm ? ((pm & (0u - pm)) << 1) - 1u : 0xffffffffu;  // up to the nearest inclusive prefix
        unsigned long long x = ((take >> tid) & 1u) ? (v & LB_VAL) : 0ull;
        for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
        excl += x;
        if (pm) break;
      }
    }
    if (tid == 0) {
      *(volatile unsigned long long *)(e.tiles + tile) = LB_PRE | (excl + agg);
      s_base = excl;
    }
  }
  if (tid < ns) s_off[tid] = off;
  __syncthreads();
  const unsigned long long base = s_base;
  if (tile + 1 == gridDim.x && tid == 0) { e.out_off[a.n_sent] = base + agg; *e.total = base + agg; }
  if (tid < ns) {
    const uint64_t s = s0 + tid;
    const unsigned long long ob = base + off;
    e.out_off[s] = ob;
    const unsigned long long first = ob + (a.reverse ? cnt - 1 : 0), last = ob + (a.reverse ? 0 : cnt - 1);
    if (a.bos) e.out[first] = a.bos_id;
    if (a.eos) e.out[last] = a.eos_id;
    if constexpr (SPANS) {
      const unsigned long long lo = a.offs[s], hi = a.offs[s + 1];
      if (a.bos) so.spans[first] = Span64{lo, lo};
      if (a.eos) so.spans[last] = Span64{hi, hi};
    }
  }
  // ---- the words' ids, EMIT_T words at a time in order: a block scan places them
  unsigned long long carry = 0;  // ids of the tile's words before the chunk
  for (uint32_t j0 = 0; j0 < n_tw; j0 += EMIT_T) {  // block-uniform
    const uint32_t j = j0 + tid;
    uint32_t k = 0, w = 0, r = 0;
    uint4 rc = make_uint4(0u, 0u, 0u, 0u);
    if (j < n_tw) {
      w = word(j, &k);
      r = rep ? rep[w] : w;
      rc = a.rec[r];
    }
    unsigned long long chunk;
    const unsigned long long x = emit_block_scan(rc.x, s_red, &chunk);
    const uint32_t n = rc.x;
    if (n) {
      // place of the word's first id in its sentence: the ids of the tile's words before it, the bos / eos of the
      // tile's sentences before it and its own bos, less the sentence's offset in the tile
      const unsigned long long p = carry + x + (unsigned long long)be * k + (a.bos ? 1 : 0) - s_off[k];
      const unsigned long long ob = base + s_off[k], last = s_ids[k] + be - 1;
      auto at = [&](unsigned long long jj) { return ob + (a.reverse ? last - jj : jj); };
      uint64_t slot = 0;
      if (SPANS || n > 3) slot = (uint64_t)a.word_pos[r] + 3ull * a.word_sent[r] + 1;
      if (n <= 3) {
        e.out[at(p)] = (int32_t)rc.y;
        if (n > 1) e.out[at(p + 1)] = (int32_t)rc.z;
        if (n > 2) e.out[at(p + 2)] = (int32_t)rc.w;
      } else {
        const int32_t *src = a.slots + slot;
        for (uint32_t q = 0; q < n; q++) e.out[at(p + q)] = src[q];
      }
      if constexpr (SPANS) {
        const unsigned long long wp = a.offs[0] + a.word_pos[w];  // this occurrence's first byte
        for (uint32_t q = 0; q < n; q++) {
          const uint2 rs = so.rel[slot + q];
          so.spans[at(p + q)] = Span64{wp + rs.x, wp + rs.y};
        }
      }
    }
    carry += chunk;
  }
}

// ---- padded output ----------------------------------------------------------------------------------------------
// encode_padded: sentence i becomes row i of an [n_sent, L] matrix instead of a run of the packed output.  With
// c = its content ids (the packed ids without <BOS> / <EOS>) and K = L - bos - eos, the row is
// [<BOS>]? c[:K] [<EOS>]?, reversed as a whole with reverse, and its cells [len, L) hold the pad id.  Row i starts at
// i L, so a tile needs nothing from the other tiles: no ticket, no look-back, no total.
//   emit_padded_kernel<SPANS, false>  a block per tile of EMIT_T consecutive sentences: content ids per sentence from
//                                     the records (a thread per word), lengths, the pad cells of the tile's rows (one
//                                     contiguous range of out), then the kept ids of every word (a thread per word)
//   emit_padded_kernel<false, true>   only the counts: the longest row of the batch (L not given)
// A word whose ids start at or past column K is skipped without reading its slots; a word that straddles the cut
// copies its kept ids only.
struct PadArgs {
  const uint32_t *rep;           // null with dropout (every word represents itself)
  int32_t *out;                  // n_sent x width
  unsigned long long *lengths;   // n_sent
  unsigned long long *max_len;   // counting form: the longest row (zeroed before the launch)
  uint64_t width;
  int32_t pad_id;
};

template <bool SPANS, bool COUNT>
__global__ void __launch_bounds__(EMIT_T) emit_padded_kernel(EncArgs a, PadArgs p, SpanOut so) {
  __shared__ uint32_t s_wb[EMIT_T];              // first work item of each sentence of the tile
  __shared__ uint32_t s_wofs[EMIT_T + 1];        // words of the tile in front of each sentence
  __shared__ uint32_t s_ids[EMIT_T];             // content ids of each sentence
  __shared__ uint32_t s_len[EMIT_T];             // row length of each sentence
  __shared__ unsigned long long s_cofs[EMIT_T];  // content ids of the tile in front of each sentence
  __shared__ unsigned long long s_red[EMIT_T / 32];
  const uint32_t tid = threadIdx.x;
  const uint64_t s0 = (uint64_t)blockIdx.x * EMIT_T;
  const uint32_t ns = (uint32_t)min((uint64_t)EMIT_T, a.n_sent - s0);
  const uint32_t be = (a.bos ? 1u : 0u) + (a.eos ? 1u : 0u);
  const uint32_t *rep = p.rep;
  s_ids[tid] = 0;
  uint32_t wc = 0;
  if (tid < ns) { s_wb[tid] = a.sent_wbase[s0 + tid]; wc = a.sent_wcnt[s0 + tid]; }
  unsigned long long tw;
  const uint32_t wofs = (uint32_t)emit_block_scan(wc, s_red, &tw);
  const uint32_t n_tw = (uint32_t)tw;  // words of the tile
  if (tid < ns) s_wofs[tid] = wofs;
  if (tid == 0) s_wofs[ns] = n_tw;
  __syncthreads();
  auto word = [&](uint32_t j, uint32_t *k) {  // the tile's j-th word: its sentence k and its work item
    uint32_t lo = 0, hi = ns;
    while (hi - lo > 1) { const uint32_t mid = (lo + hi) >> 1; if (s_wofs[mid] <= j) lo = mid; else hi = mid; }
    *k = lo;
    return s_wb[lo] + (j - s_wofs[lo]);
  };
  for (uint32_t j = tid; j < n_tw; j += EMIT_T) {
    uint32_t k;
    const uint32_t w = word(j, &k);
    atomicAdd(&s_ids[k], a.rec[rep ? rep[w] : w].x);
  }
  __syncthreads();
  const uint32_t cnt = tid < ns ? s_ids[tid] : 0u;
  if constexpr (COUNT) {
    unsigned long long m = tid < ns ? (unsigned long long)cnt + be : 0ull;
    for (int o = 16; o > 0; o >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((tid & 31) == 0) s_red[tid >> 5] = m;
    __syncthreads();
    if (tid == 0) {
      for (int i = 1; i < EMIT_T / 32; i++) m = max(m, s_red[i]);
      atomicMax(p.max_len, m);
    }
    return;
  }
  const uint64_t L = p.width, K = L - be;  // L >= bos + eos (checked by the host)
  const uint32_t len = tid < ns ? (uint32_t)(min((uint64_t)cnt, K) + be) : 0u;
  unsigned long long tot;
  const unsigned long long cofs = emit_block_scan(cnt, s_red, &tot);
  if (tid < ns) {
    const uint64_t s = s0 + tid;
    s_cofs[tid] = cofs;
    s_len[tid] = len;
    p.lengths[s] = len;
    if (len) {
      const uint64_t row = s * L, first = row + (a.reverse ? len - 1 : 0), last = row + (a.reverse ? 0 : len - 1);
      if (a.bos) p.out[first] = a.bos_id;
      if (a.eos) p.out[last] = a.eos_id;
      if constexpr (SPANS) {
        const unsigned long long lo = a.offs[s], hi = a.offs[s + 1];
        if (a.bos) so.spans[first] = Span64{lo, lo};
        if (a.eos) so.spans[last] = Span64{hi, hi};
      }
    }
  }
  __syncthreads();
  // ---- the pad cells: the tile's rows are the cells [s0 L, (s0 + ns) L) of out; thread t takes cells t, t + EMIT_T,
  // ... and steps its (row, column) without a division per cell
  if (L) {
    const uint64_t n_cells = (uint64_t)ns * L, step_r = EMIT_T / L, step_c = EMIT_T % L;
    uint64_t r = tid / L, col = tid % L;
    int32_t *out = p.out + s0 * L;
    for (uint64_t x = tid; x < n_cells; x += EMIT_T) {
      if (col >= s_len[r]) {
        out[x] = p.pad_id;
        if constexpr (SPANS) {
          const unsigned long long hi = a.offs[s0 + r + 1];
          so.spans[s0 * L + x] = Span64{hi, hi};
        }
      }
      r += step_r;
      col += step_c;
      if (col >= L) { col -= L; r++; }
    }
  }
  // ---- the words' kept ids, EMIT_T words at a time in order: a block scan gives each word its first content index
  unsigned long long carry = 0;  // content ids of the tile's words before the chunk
  for (uint32_t j0 = 0; j0 < n_tw; j0 += EMIT_T) {  // block-uniform
    const uint32_t j = j0 + tid;
    uint32_t k = 0, w = 0, r = 0;
    uint4 rc = make_uint4(0u, 0u, 0u, 0u);
    if (j < n_tw) {
      w = word(j, &k);
      r = rep ? rep[w] : w;
      rc = a.rec[r];
    }
    unsigned long long chunk;
    const unsigned long long x = emit_block_scan(rc.x, s_red, &chunk);
    const uint32_t n = rc.x;
    const unsigned long long c0 = carry + x - (n ? s_cofs[k] : 0ull);  // the word's first content index in its row
    if (n && c0 < K) {
      const uint32_t m = (uint32_t)min((unsigned long long)n, K - c0);  // ids of the word that are kept
      const uint64_t row = (s0 + k) * L, last = s_len[k] - 1, c1 = c0 + (a.bos ? 1 : 0);
      auto at = [&](uint32_t q) { return row + (a.reverse ? last - (c1 + q) : c1 + q); };
      uint64_t slot = 0;
      if (SPANS || n > 3) slot = (uint64_t)a.word_pos[r] + 3ull * a.word_sent[r] + 1;
      if (n <= 3) {
        p.out[at(0)] = (int32_t)rc.y;
        if (m > 1) p.out[at(1)] = (int32_t)rc.z;
        if (m > 2) p.out[at(2)] = (int32_t)rc.w;
      } else {
        const int32_t *src = a.slots + slot;
        for (uint32_t q = 0; q < m; q++) p.out[at(q)] = src[q];
      }
      if constexpr (SPANS) {
        const unsigned long long wp = a.offs[0] + a.word_pos[w];  // this occurrence's first byte
        for (uint32_t q = 0; q < m; q++) {
          const uint2 rs = so.rel[slot + q];
          so.spans[at(q)] = Span64{wp + rs.x, wp + rs.y};
        }
      }
    }
    carry += chunk;
  }
}

// ---- subwords ---------------------------------------------------------------------------------------------------
// One piece per output id: the model's piece of an ordinary id (recipe UTF-8, leading U+2581 kept) or of <BOS> / <EOS>,
// and for <UNK> the characters of its run: the valid units of its span, copied from the source bytes.
struct SubArgs {
  const int32_t *ids;
  const Span64 *spans;
  uint64_t n;                  // ids
  const uint8_t *bytes;        // batch bytes; span value v is batch byte v - offs[0]
  const uint64_t *offs;
  const uint32_t *piece_off;   // V + 1
  const uint8_t *piece_bytes;
  int32_t unk_id;
};

__global__ void __launch_bounds__(256) sub_count_kernel(SubArgs a, unsigned long long *__restrict__ len) {
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  const uint64_t o0 = a.offs[0];
  for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j < a.n; j += stride) {
    const int32_t id = a.ids[j];
    if (id != a.unk_id) { len[j] = __ldg(a.piece_off + id + 1) - __ldg(a.piece_off + id); continue; }
    const Span64 sp = a.spans[j];
    unsigned long long m = 0;
    uint32_t l;
    for (uint64_t q = sp.lo - o0, e = sp.hi - o0; q < e; q += l)
      if (decode_unit(a.bytes, q, e, &l) != INVALID_CP) m += l;
    len[j] = m;
  }
}

__global__ void __launch_bounds__(256) sub_emit_kernel(SubArgs a, const unsigned long long *__restrict__ off,
                                                       uint8_t *__restrict__ out) {
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  const uint64_t o0 = a.offs[0];
  for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j < a.n; j += stride) {
    const int32_t id = a.ids[j];
    uint8_t *dst = out + off[j];
    if (id != a.unk_id) {
      const uint32_t b = __ldg(a.piece_off + id), e = __ldg(a.piece_off + id + 1);
      for (uint32_t k = b; k < e; k++) *dst++ = __ldg(a.piece_bytes + k);
      continue;
    }
    const Span64 sp = a.spans[j];
    uint32_t l;
    for (uint64_t q = sp.lo - o0, e = sp.hi - o0; q < e; q += l)
      if (decode_unit(a.bytes, q, e, &l) != INVALID_CP)
        for (uint32_t k = 0; k < l; k++) *dst++ = a.bytes[q + k];
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

// what an encode call computes: ids; ids + spans; ids + spans + subword pieces
enum EncMode { ENC_IDS = 0, ENC_SPANS = 1, ENC_SUBWORDS = 2 };

// The subword piece and the unit count of every id, one upload (the first spans / subwords call of an encoder).
int build_sub_table(yttm_enc *e) {
  yttm_ctx *c = e->ctx;
  const uint64_t V = e->vocab;
  std::vector<std::string> raw;
  std::vector<uint8_t> special;
  if (yttm_model_pieces(e, "encode", &raw, &special)) return 1;
  std::vector<uint32_t> head(2 * V + 1);  // piece_off[V + 1] | units[V]
  uint64_t total = 0;
  for (uint64_t i = 0; i < V; i++) {
    head[i] = (uint32_t)total;
    total += raw[i].size();
    if (total > 0xffffff00ull) YT_FAIL(c, "encode: piece table over 4 GB");
    uint32_t u = 0;
    if (!special[i]) {
      for (unsigned char b : raw[i]) u += (b & 0xc0) != 0x80;  // code points of valid UTF-8
      if (raw[i].compare(0, 3, "\xe2\x96\x81") == 0) u -= 1;    // the word-initial U+2581 covers no unit
    }
    head[V + 1 + i] = u;
  }
  head[V] = (uint32_t)total;
  const uint64_t a_bytes = ((2 * V + 1) * 4 + 15) & ~15ull, size = a_bytes + total + 16;
  std::vector<uint8_t> h(size, 0);
  std::memcpy(h.data(), head.data(), head.size() * 4);
  for (uint64_t i = 0; i < V; i++) std::memcpy(h.data() + a_bytes + head[i], raw[i].data(), raw[i].size());
  YT_CUDA(c, e->sub_table.reserve(size));
  YT_CUDA(c, cudaMemcpyAsync(e->sub_table.p, h.data(), size, cudaMemcpyHostToDevice, c->stream));
  YT_CUDA(c, cudaStreamSynchronize(c->stream));
  e->sub_piece_off = e->sub_table.as<uint32_t>();
  e->sub_units = e->sub_piece_off + V + 1;
  e->sub_bytes = e->sub_table.as<uint8_t>() + a_bytes;
  return 0;
}

// The padded form of an encode call: rows of `width` ids (0 = the longest row of the batch, set by enc_device).
struct PadReq {
  uint64_t width;
  int32_t pad_id;
};

// Encodes one batch on the device.  mode >= ENC_SPANS also writes e->out_spans; ENC_SUBWORDS also the pieces
// (e->sub_off: out_n + 1 byte offsets, e->sub_out: *out_bytes bytes).  With pad (ENC_IDS / ENC_SPANS) the ids and
// spans are the n_sent x pad->width rows of emit_padded_kernel and e->out_off holds the row lengths.
int enc_device(yttm_enc *enc, yttm_enc::Slot *e, const uint8_t *d_bytes, const uint64_t *d_offs, uint64_t n_bytes,
               uint64_t n_sent, int bos, int eos, int reverse, double dropout, uint64_t seed, uint64_t first_sentence,
               uint64_t *out_n, int mode = ENC_IDS, uint64_t *out_bytes = nullptr, PadReq *pad = nullptr) {
  yttm_ctx *c = enc->ctx;
  if (n_bytes >= 0xfffffff0ull || n_sent >= 0xfffffff0ull)
    YT_FAIL(c, "encode batch too large: at most 2^32 bytes / sentences per call (split the batch)");
  const uint64_t n_slots = n_bytes + 3 * n_sent;
  if (out_bytes) *out_bytes = 0;
  SpanOut so{nullptr, nullptr, nullptr};
  if (mode != ENC_IDS) {
    if (!enc->sub_piece_off && build_sub_table(enc)) return 1;
    YT_CUDA(c, e->rel.reserve((n_slots + 8) * 8));
    so.rel = e->rel.as<uint2>();
    so.units = enc->sub_units;
  }
  YT_CUDA(c, e->slots.reserve((n_slots + 8) * 4));
  YT_CUDA(c, e->ranks.reserve((n_slots + 8) * 4));
  if (dropout > 0) YT_CUDA(c, e->aux.reserve((n_slots + 8) * 24));
  const uint64_t max_words = n_bytes / 2 + n_sent + 8;
  YT_CUDA(c, e->wpos.reserve(max_words * 4));
  YT_CUDA(c, e->wsent.reserve(max_words * 4));
  const uint64_t n_tiles = (n_sent + EMIT_T - 1) / EMIT_T;
  YT_CUDA(c, e->lookback.reserve((n_tiles + 1) * 8));
  YT_CUDA(c, e->out_off.reserve((n_sent + 2) * 8));
  YT_CUDA(c, e->counter.reserve(64));
  YT_CUDA(c, cudaMemsetAsync(e->counter.p, 0, 64, c->stream));
  EncArgs a;
  a.bytes = d_bytes; a.offs = d_offs; a.n_sent = n_sent;
  a.slots = e->slots.as<int32_t>(); a.ranks = e->ranks.as<uint32_t>();
  a.aux = dropout > 0 ? e->aux.as<uint32_t>() : nullptr;
  a.word_pos = e->wpos.as<uint32_t>(); a.word_sent = e->wsent.as<uint32_t>();
  a.n_words = e->counter.as<unsigned long long>();
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
  a.rec = nullptr;  // sized by the number of words, known after find_words_vec_kernel
  {
    ytc::timer_begin(c, "enc_find");
    // sentences per group: a group of mean-length sentences fills about 3/4 of a piece, so that groups longer than a
    // piece (two passes) stay rare
    const uint64_t mean = std::max<uint64_t>(n_bytes / n_sent, 1);
    const uint32_t G = (uint32_t)std::min<uint64_t>(FIND_GMAX, std::max<uint64_t>(FIND_TILE * 3 / 4 / mean, 1));
    const uint64_t blocks = std::min<uint64_t>((n_sent + G - 1) / G, (uint64_t)c->n_sm * 4);
    find_words_vec_kernel<<<(unsigned)std::max<uint64_t>(blocks, 1), FIND_T, 0, c->stream>>>(a, G);
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
    YT_CUDA(c, e->rec.reserve(n_words * 16 + 16));
    a.rec = e->rec.as<uint4>();
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
      if (const int v = ytc::env_int("YTTM_ENC_DEDUP_SLOTS", 0, 1, INT_MAX)) tslots = ytc::pow2ceil((uint64_t)v);  // tests: tiny tables
      YT_CUDA(c, e->dd_tab.reserve(tslots * 8));
      YT_CUDA(c, e->dd_rep.reserve(n_words * 4 + 16));
      YT_CUDA(c, e->dd_list.reserve(n_words * 4 + 16));
      DedupArgs d;
      d.tab = e->dd_tab.as<unsigned long long>(); d.mask = (uint32_t)(tslots - 1);
      d.rep = e->dd_rep.as<uint32_t>(); d.list = e->dd_list.as<uint32_t>();
      d.n_list = e->counter.as<unsigned long long>() + 2;  // zeroed with the other counters above
      d.weak_tag = ytc::env_set("YTTM_ENC_DEDUP_WEAKTAG");  // tests: tag collisions everywhere
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
      if (mode != ENC_IDS) {
        ytc::timer_begin(c, "enc_spans");
        span_words_kernel<<<(unsigned)blocks, 128, 0, c->stream>>>(a, d.list, d.n_list, 0, so);
        ytc::timer_end(c, "enc_spans");
        c->launches++;
      }
    } else {
      encode_words_kernel<<<(unsigned)blocks, 128, 0, c->stream>>>(a, n_words);
      c->launches++;
      if (mode != ENC_IDS) {
        ytc::timer_begin(c, "enc_spans");
        span_words_kernel<<<(unsigned)blocks, 128, 0, c->stream>>>(a, nullptr, nullptr, n_words, so);
        ytc::timer_end(c, "enc_spans");
        c->launches++;
      }
    }
    ytc::timer_end(c, "enc_words");
  }
  if (pad) {  // rows of width L: n_sent x L ids (and spans) are reserved, not the packed bound
    PadArgs pa;
    pa.rep = d_rep; pa.lengths = e->out_off.as<unsigned long long>(); pa.max_len = d_total; pa.pad_id = pad->pad_id;
    pa.out = nullptr; pa.width = 0;
    const unsigned n_tiles_pad = (unsigned)n_tiles;
    ytc::timer_begin(c, "enc_gather");
    if (pad->width == 0) {  // the longest row: one counting pass and one 8-byte read-back (d_total was zeroed above)
      emit_padded_kernel<false, true><<<n_tiles_pad, EMIT_T, 0, c->stream>>>(a, pa, so);
      c->launches++;
      unsigned long long longest = 0;
      YT_CUDA(c, cudaMemcpyAsync(&longest, d_total, 8, cudaMemcpyDeviceToHost, c->stream));
      YT_CUDA(c, cudaStreamSynchronize(c->stream));
      if (longest > 0x7fffffffull) YT_FAIL(c, "encode padded: the longest row has more than 2^31 - 1 ids (pass a width)");
      pad->width = longest;
    }
    const uint64_t cells = n_sent * pad->width;  // < 2^32 * 2^31
    const uint64_t span_bytes = mode != ENC_IDS ? cells * 16 : 0;
    if (cells > (1ull << 40) || e->out_ids.reserve(cells * 4 + 16) != cudaSuccess ||
        (span_bytes && e->out_spans.reserve(span_bytes + 16) != cudaSuccess)) {
      cudaGetLastError();  // the failed allocation is reported here, not by the next call
      YT_FAIL(c, "encode padded: " + std::to_string(n_sent) + " x " + std::to_string(pad->width) +
                     " rows do not fit in device memory (split the batch or lower the width)");
    }
    pa.out = e->out_ids.as<int32_t>(); pa.width = pad->width;
    if (mode != ENC_IDS) so.spans = e->out_spans.as<Span64>();
    if (mode == ENC_IDS) emit_padded_kernel<false, false><<<n_tiles_pad, EMIT_T, 0, c->stream>>>(a, pa, so);
    else emit_padded_kernel<true, false><<<n_tiles_pad, EMIT_T, 0, c->stream>>>(a, pa, so);
    c->launches++;
    ytc::timer_end(c, "enc_gather");
    ytc::timer_end(c, "encode");
    YT_CUDA(c, cudaGetLastError());
    *out_n = cells;
    return 0;
  }
  // The output is reserved at a bound, so that the emit needs no count from the host first: a sentence of len bytes
  // has at most len + 1 + bos + eos ids (a word of k bytes has at most k + 1 ids, and its words are separated by at least
  // one byte each).
  const uint64_t id_cap = n_bytes + (1ull + (bos ? 1 : 0) + (eos ? 1 : 0)) * n_sent;
  YT_CUDA(c, e->out_ids.reserve((id_cap + 8) * 4));
  if (mode != ENC_IDS) {
    YT_CUDA(c, e->out_spans.reserve((id_cap + 8) * 16));
    so.spans = e->out_spans.as<Span64>();
  }
  YT_CUDA(c, cudaMemsetAsync(e->lookback.p, 0, n_tiles * 8, c->stream));
  EmitArgs ea;
  ea.rep = d_rep; ea.tiles = e->lookback.as<unsigned long long>();
  ea.ticket = e->counter.as<unsigned long long>() + 3;  // zeroed with the other counters above
  ea.total = d_total; ea.out_off = e->out_off.as<unsigned long long>(); ea.out = e->out_ids.as<int32_t>();
  ytc::timer_begin(c, "enc_gather");
  if (mode == ENC_IDS) emit_ids_kernel<false><<<(unsigned)n_tiles, EMIT_T, 0, c->stream>>>(a, ea, so);
  else emit_ids_kernel<true><<<(unsigned)n_tiles, EMIT_T, 0, c->stream>>>(a, ea, so);
  ytc::timer_end(c, "enc_gather");
  c->launches++;
  unsigned long long total = 0;
  YT_CUDA(c, cudaMemcpyAsync(&total, d_total, 8, cudaMemcpyDeviceToHost, c->stream));
  YT_CUDA(c, cudaStreamSynchronize(c->stream));
  if (mode == ENC_SUBWORDS && total == 0) {
    YT_CUDA(c, e->sub_off.reserve(16));
    YT_CUDA(c, cudaMemsetAsync(e->sub_off.p, 0, 8, c->stream));
  } else if (mode == ENC_SUBWORDS) {  // piece lengths -> exclusive scan -> piece bytes
    SubArgs sa;
    sa.ids = e->out_ids.as<int32_t>(); sa.spans = so.spans; sa.n = total;
    sa.bytes = d_bytes; sa.offs = d_offs;
    sa.piece_off = enc->sub_piece_off; sa.piece_bytes = enc->sub_bytes; sa.unk_id = enc->unk;
    YT_CUDA(c, e->sub_len.reserve((total + 8) * 8));
    YT_CUDA(c, e->sub_off.reserve((total + 8) * 8));
    unsigned long long *sub_off = e->sub_off.as<unsigned long long>();
    const uint64_t iblocks = std::max<uint64_t>(std::min<uint64_t>((total + 255) / 256, (uint64_t)c->n_sm * 8), 1);
    ytc::timer_begin(c, "enc_subwords");
    sub_count_kernel<<<(unsigned)iblocks, 256, 0, c->stream>>>(sa, e->sub_len.as<unsigned long long>());
    c->launches++;
    if (yttm_device_scan_u64(c, e->sub_len.as<unsigned long long>(), total, sub_off, d_total)) return 1;
    unsigned long long n_piece_bytes = 0;
    YT_CUDA(c, cudaMemcpyAsync(&n_piece_bytes, d_total, 8, cudaMemcpyDeviceToHost, c->stream));
    YT_CUDA(c, cudaMemcpyAsync(sub_off + total, d_total, 8, cudaMemcpyDeviceToDevice, c->stream));
    YT_CUDA(c, cudaStreamSynchronize(c->stream));
    YT_CUDA(c, e->sub_out.reserve(n_piece_bytes + 16));
    sub_emit_kernel<<<(unsigned)iblocks, 256, 0, c->stream>>>(sa, sub_off, e->sub_out.as<uint8_t>());
    c->launches++;
    ytc::timer_end(c, "enc_subwords");
    *out_bytes = n_piece_bytes;
  }
  ytc::timer_end(c, "encode");
  YT_CUDA(c, cudaGetLastError());
  *out_n = total;
  return 0;
}

// Caller buffers of the host-buffer entry points; nullptr = not asked for.  ids_cap bounds ids / spans / pieces (one
// piece per id), bytes_cap the piece bytes.
struct HostOut {
  int mode;
  int32_t *ids;
  uint64_t *spans;              // 2 per id
  uint64_t ids_cap;
  uint64_t *id_offsets;         // n_sent + 1
  uint8_t *pieces;
  uint64_t bytes_cap;
  uint64_t *piece_offsets;      // n_pieces + 1
  const PadReq *pad = nullptr;  // padded rows: ids / spans hold n_sent x pad->width cells
  uint64_t *lengths = nullptr;  // padded rows: n_sent
};

// The host-buffer form of enc_device: the batch is cut into chunks at sentence boundaries, chunk i runs in slot i & 1
// while the copies of its neighbours overlap it.  Returns 2 with *out_n / *out_bytes = the sizes needed when a capacity
// is too small.
int enc_run_host(yttm_enc *e, const char *who, const char *bytes, const uint64_t *offsets, uint64_t n_sent, int bos,
                 int eos, int reverse, double dropout, uint64_t seed, uint64_t first_sentence_index, const HostOut &o,
                 uint64_t *out_n, uint64_t *out_bytes) {
  yttm_ctx *c = e->ctx;
  *out_n = 0;
  if (out_bytes) *out_bytes = 0;
  if (n_sent == 0) {
    if (o.id_offsets) o.id_offsets[0] = 0;
    if (o.piece_offsets) o.piece_offsets[0] = 0;
    return 0;
  }
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
  const uint64_t chunk_bytes = (uint64_t)ytc::env_int("YTTM_ENC_CHUNK_MB", 32, 1, INT_MAX) << 20;
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
  c->enc_chunks = (double)K;  // yttm_stage_ms(ctx, "enc_chunks"): how many chunks the last host-buffer call used
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
  uint64_t base = 0, bbase = 0;  // ids / piece bytes of the chunks before
  int rc_small = 0;
  for (size_t i = 0; i < K; i++) {
    yttm_enc::Slot &sl = e->slot[i & 1];
    const uint64_t lo = cut[i], hi = cut[i + 1], nb = offsets[hi] - offsets[lo];
    if (i + 1 < K && h2d(i + 1)) return 1;
    YT_CUDA(c, cudaStreamWaitEvent(c->stream, e->ev_in[i & 1], 0));
    if (i >= 2) YT_CUDA(c, cudaStreamWaitEvent(c->stream, e->ev_out[i & 1], 0));  // results of chunk i-2 have left
    uint64_t total = 0, tbytes = 0;
    PadReq pr{0, 0};
    if (o.pad) pr = *o.pad;
    if (enc_device(e, &sl, sl.d_bytes.as<uint8_t>(), sl.d_offs.as<uint64_t>(), nb, hi - lo, bos, eos, reverse, dropout,
                   seed, first_sentence_index + lo, &total, o.mode, &tbytes, o.pad ? &pr : nullptr))
      return 1;
    if (o.pad) {  // rows [lo, hi) land at row lo: nothing to rebase
      const uint64_t W = pr.width;
      YT_CUDA(c, cudaEventRecord(e->ev_done[i & 1], c->stream));
      YT_CUDA(c, cudaStreamWaitEvent(e->s_out, e->ev_done[i & 1], 0));
      YT_CUDA(c, cudaMemcpyAsync(o.ids + lo * W, sl.out_ids.p, (hi - lo) * W * 4, cudaMemcpyDeviceToHost, e->s_out));
      if (o.spans)
        YT_CUDA(c, cudaMemcpyAsync(o.spans + 2 * lo * W, sl.out_spans.p, (hi - lo) * W * 16, cudaMemcpyDeviceToHost, e->s_out));
      YT_CUDA(c, cudaMemcpyAsync(o.lengths + lo, sl.out_off.p, (hi - lo) * 8, cudaMemcpyDeviceToHost, e->s_out));
      YT_CUDA(c, cudaEventRecord(e->ev_out[i & 1], e->s_out));
      base += total;
      continue;
    }
    if (base && hi > lo) {  // chunk-local offsets -> batch offsets
      add_base_kernel<<<(unsigned)std::min<uint64_t>((hi - lo + 255) / 256, (uint64_t)c->n_sm * 4), 256, 0, c->stream>>>(
          sl.out_off.as<unsigned long long>(), hi - lo, (unsigned long long)base);
      c->launches++;
    }
    if (o.piece_offsets && bbase && total) {  // the same for the piece offsets (spans are batch coordinates already)
      add_base_kernel<<<(unsigned)std::min<uint64_t>((total + 255) / 256, (uint64_t)c->n_sm * 4), 256, 0, c->stream>>>(
          sl.sub_off.as<unsigned long long>(), total, (unsigned long long)bbase);
      c->launches++;
    }
    YT_CUDA(c, cudaEventRecord(e->ev_done[i & 1], c->stream));
    if (base + total > o.ids_cap || bbase + tbytes > o.bytes_cap) rc_small = 2;
    if (!rc_small) {
      YT_CUDA(c, cudaStreamWaitEvent(e->s_out, e->ev_done[i & 1], 0));
      if (total && o.ids)
        YT_CUDA(c, cudaMemcpyAsync(o.ids + base, sl.out_ids.p, total * 4, cudaMemcpyDeviceToHost, e->s_out));
      if (total && o.spans)
        YT_CUDA(c, cudaMemcpyAsync(o.spans + 2 * base, sl.out_spans.p, total * 16, cudaMemcpyDeviceToHost, e->s_out));
      if (total && o.piece_offsets)
        YT_CUDA(c, cudaMemcpyAsync(o.piece_offsets + base, sl.sub_off.p, total * 8, cudaMemcpyDeviceToHost, e->s_out));
      if (tbytes && o.pieces)
        YT_CUDA(c, cudaMemcpyAsync(o.pieces + bbase, sl.sub_out.p, tbytes, cudaMemcpyDeviceToHost, e->s_out));
      YT_CUDA(c, cudaMemcpyAsync(o.id_offsets + lo, sl.out_off.p, (hi - lo) * 8, cudaMemcpyDeviceToHost, e->s_out));
      YT_CUDA(c, cudaEventRecord(e->ev_out[i & 1], e->s_out));
    }
    base += total;
    bbase += tbytes;
  }
  YT_CUDA(c, cudaStreamSynchronize(e->s_out));
  YT_CUDA(c, cudaStreamSynchronize(c->stream));
  ytc::timer_end(c, "e2e");
  *out_n = base;
  if (out_bytes) *out_bytes = bbase;
  if (rc_small) { c->err = std::string(who) + ": output buffer too small"; return 2; }
  if (o.id_offsets) o.id_offsets[n_sent] = base;
  if (o.piece_offsets) o.piece_offsets[base] = bbase;
  (void)total_bytes;
  return 0;
}

// The epilogue of the device entry points: every output buffer is allocated (the pointers handed out are never null),
// the offsets of an empty batch read [0], and the stream is idle, so that readers on any stream see complete results.
int publish_device(yttm_ctx *c, uint64_t n_sent, std::initializer_list<ytc::DevBuf *> outs,
                   std::initializer_list<ytc::DevBuf *> offsets) {
  for (ytc::DevBuf *b : outs) YT_CUDA(c, b->reserve(16));
  for (ytc::DevBuf *b : offsets) {
    YT_CUDA(c, b->reserve(16));
    if (n_sent == 0) YT_CUDA(c, cudaMemsetAsync(b->p, 0, 8, c->stream));
  }
  YT_CUDA(c, cudaStreamSynchronize(c->stream));
  return 0;
}

}  // namespace

int yttm_enc_check(yttm_enc *e, const char *who, int bos, int eos) {
  if (!e) {
    g_yttm_create_error = std::string(who) + ": null encoder handle (no CUDA device, or yttm_enc_create failed)";
    return 1;
  }
  yttm_ctx *c = e->ctx;
  YT_CUDA(c, cudaSetDevice(c->device));
  ytc::timers_reset(c);   // every encode and decode call starts here: the stage times describe this call alone
  if (bos && e->bos == -1) YT_FAIL(c, "Can't add <BOS> token. Model was trained without it.");
  if (eos && e->eos == -1) YT_FAIL(c, "Can't add <EOS> token. Model was trained without it.");
  return 0;
}

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
  e->sub_table.release();
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
  if (yttm_enc_check(e, "yttm_enc_run_device", bos, eos)) return 1;
  yttm_enc::Slot &sl = e->slot[0];
  if (enc_device(e, &sl, (const uint8_t *)d_bytes, d_offsets, n_bytes, n_sent, bos, eos, reverse, dropout, seed,
                 first_sentence_index, out_n) ||
      publish_device(e->ctx, n_sent, {&sl.out_ids}, {&sl.out_off}))
    return 1;
  if (d_out_ids) *d_out_ids = sl.out_ids.as<int32_t>();
  if (d_out_offsets) *d_out_offsets = sl.out_off.as<uint64_t>();
  return 0;
}

int yttm_enc_run(yttm_enc *e, const char *bytes, const uint64_t *offsets, uint64_t n_sent, int bos, int eos, int reverse,
                 double dropout, uint64_t seed, uint64_t first_sentence_index, int32_t *out_ids, uint64_t out_cap,
                 uint64_t *out_offsets, uint64_t *out_n) {
  if (yttm_enc_check(e, "yttm_enc_run", bos, eos)) return 1;
  const HostOut o{ENC_IDS, out_ids, nullptr, out_cap, out_offsets, nullptr, ~0ull, nullptr};
  return enc_run_host(e, "yttm_enc_run", bytes, offsets, n_sent, bos, eos, reverse, dropout, seed, first_sentence_index, o,
                      out_n, nullptr);
}

int yttm_enc_run_spans_device(yttm_enc *e, const char *d_bytes, const uint64_t *d_offsets, uint64_t n_bytes, uint64_t n_sent,
                              int bos, int eos, int reverse, double dropout, uint64_t seed, uint64_t first_sentence_index,
                              const int32_t **d_out_ids, const uint64_t **d_out_offsets, const uint64_t **d_out_spans,
                              uint64_t *out_n) {
  if (yttm_enc_check(e, "yttm_enc_run_spans_device", bos, eos)) return 1;
  yttm_enc::Slot &sl = e->slot[0];
  if (enc_device(e, &sl, (const uint8_t *)d_bytes, d_offsets, n_bytes, n_sent, bos, eos, reverse, dropout, seed,
                 first_sentence_index, out_n, ENC_SPANS) ||
      publish_device(e->ctx, n_sent, {&sl.out_ids, &sl.out_spans}, {&sl.out_off}))
    return 1;
  if (d_out_ids) *d_out_ids = sl.out_ids.as<int32_t>();
  if (d_out_offsets) *d_out_offsets = sl.out_off.as<uint64_t>();
  if (d_out_spans) *d_out_spans = sl.out_spans.as<uint64_t>();
  return 0;
}

int yttm_enc_run_spans(yttm_enc *e, const char *bytes, const uint64_t *offsets, uint64_t n_sent, int bos, int eos,
                       int reverse, double dropout, uint64_t seed, uint64_t first_sentence_index, int32_t *out_ids,
                       uint64_t out_cap, uint64_t *out_offsets, uint64_t *out_spans, uint64_t *out_n) {
  if (yttm_enc_check(e, "yttm_enc_run_spans", bos, eos)) return 1;
  const HostOut o{ENC_SPANS, out_ids, out_spans, out_cap, out_offsets, nullptr, ~0ull, nullptr};
  return enc_run_host(e, "yttm_enc_run_spans", bytes, offsets, n_sent, bos, eos, reverse, dropout, seed,
                      first_sentence_index, o, out_n, nullptr);
}

int yttm_enc_run_padded(yttm_enc *e, const char *bytes, const uint64_t *offsets, uint64_t n_sent, int bos, int eos,
                        int reverse, double dropout, uint64_t seed, uint64_t first_sentence_index, uint64_t width,
                        int32_t pad_id, int32_t *out_ids, uint64_t *out_lengths, uint64_t *out_spans) {
  if (yttm_enc_check(e, "yttm_enc_run_padded", bos, eos)) return 1;
  if (width == 0 || width < (uint64_t)(bos ? 1 : 0) + (eos ? 1 : 0) || width > 0x7fffffffull)
    YT_FAIL(e->ctx, "yttm_enc_run_padded: width must be at least 1 and bos + eos, and below 2^31");
  PadReq pr{width, pad_id};
  HostOut o{out_spans ? ENC_SPANS : ENC_IDS, out_ids, out_spans, ~0ull, nullptr, nullptr, ~0ull, nullptr, &pr, out_lengths};
  uint64_t n = 0;
  return enc_run_host(e, "yttm_enc_run_padded", bytes, offsets, n_sent, bos, eos, reverse, dropout, seed,
                      first_sentence_index, o, &n, nullptr);
}

int yttm_enc_run_padded_device(yttm_enc *e, const char *d_bytes, const uint64_t *d_offsets, uint64_t n_bytes,
                               uint64_t n_sent, int bos, int eos, int reverse, double dropout, uint64_t seed,
                               uint64_t first_sentence_index, uint64_t width, int32_t pad_id, int with_spans,
                               const int32_t **d_ids, const uint64_t **d_lengths, const uint64_t **d_spans,
                               uint32_t *out_width) {
  if (yttm_enc_check(e, "yttm_enc_run_padded_device", bos, eos)) return 1;
  if (width && (width < (uint64_t)(bos ? 1 : 0) + (eos ? 1 : 0) || width > 0x7fffffffull))
    YT_FAIL(e->ctx, "yttm_enc_run_padded_device: width must be 0 (the longest row) or at least bos + eos, and below 2^31");
  yttm_enc::Slot &sl = e->slot[0];
  PadReq pr{width, pad_id};
  uint64_t n = 0;
  if (enc_device(e, &sl, (const uint8_t *)d_bytes, d_offsets, n_bytes, n_sent, bos, eos, reverse, dropout, seed,
                 first_sentence_index, &n, with_spans ? ENC_SPANS : ENC_IDS, nullptr, &pr) ||
      publish_device(e->ctx, n_sent, {&sl.out_ids, &sl.out_spans}, {&sl.out_off}))
    return 1;
  if (d_ids) *d_ids = sl.out_ids.as<int32_t>();
  if (d_lengths) *d_lengths = sl.out_off.as<uint64_t>();
  if (d_spans) *d_spans = with_spans ? sl.out_spans.as<uint64_t>() : nullptr;
  if (out_width) *out_width = (uint32_t)pr.width;
  return 0;
}

int yttm_enc_run_subwords_device(yttm_enc *e, const char *d_bytes, const uint64_t *d_offsets, uint64_t n_bytes,
                                 uint64_t n_sent, int bos, int eos, int reverse, double dropout, uint64_t seed,
                                 uint64_t first_sentence_index, const uint8_t **d_pieces, const uint64_t **d_piece_offsets,
                                 const uint64_t **d_sent_offsets, uint64_t *n_pieces, uint64_t *n_piece_bytes) {
  if (yttm_enc_check(e, "yttm_enc_run_subwords_device", bos, eos)) return 1;
  yttm_enc::Slot &sl = e->slot[0];
  if (enc_device(e, &sl, (const uint8_t *)d_bytes, d_offsets, n_bytes, n_sent, bos, eos, reverse, dropout, seed,
                 first_sentence_index, n_pieces, ENC_SUBWORDS, n_piece_bytes) ||
      publish_device(e->ctx, n_sent, {&sl.sub_out}, {&sl.out_off, &sl.sub_off}))
    return 1;
  if (d_pieces) *d_pieces = sl.sub_out.as<uint8_t>();
  if (d_piece_offsets) *d_piece_offsets = sl.sub_off.as<uint64_t>();
  if (d_sent_offsets) *d_sent_offsets = sl.out_off.as<uint64_t>();
  return 0;
}

int yttm_enc_run_subwords(yttm_enc *e, const char *bytes, const uint64_t *offsets, uint64_t n_sent, int bos, int eos,
                          int reverse, double dropout, uint64_t seed, uint64_t first_sentence_index, uint8_t *out_pieces,
                          uint64_t bytes_cap, uint64_t *out_piece_offsets, uint64_t pieces_cap, uint64_t *out_sent_offsets,
                          uint64_t *n_pieces, uint64_t *n_piece_bytes) {
  if (yttm_enc_check(e, "yttm_enc_run_subwords", bos, eos)) return 1;
  const HostOut o{ENC_SUBWORDS, nullptr, nullptr, pieces_cap, out_sent_offsets, out_pieces, bytes_cap, out_piece_offsets};
  return enc_run_host(e, "yttm_enc_run_subwords", bytes, offsets, n_sent, bos, eos, reverse, dropout, seed,
                      first_sentence_index, o, n_pieces, n_piece_bytes);
}
}  // extern "C"
