// merge_loop.cuh — phase 4 of training: the persistent merge loop (included by train.cu).
//
// Replaces the reference's main loop + worker_doing_merge + PriorityQueue
// (bpe.cpp:1121-1282, 601-811, 149-314) and, across GPUs, the per-merge count exchange between
// its worker threads (check_cnt :1099-1108, workers reporting the pairs of the new token :789-804,
// main gathering them :1239-1266).  One cooperative kernel per GPU runs every merge iteration on
// the device.  Design (round 2, "owner computes"):
//   * the pair table is cut into one PARTITION per block (PairTab::nparts == gridDim.x); block b
//     is the only one that ever reads or writes partition b inside the loop;
//   * a block never touches the table while it rewrites words: the count changes of a merge
//     (key, +-delta) are appended to the block's own SEGMENT of an exchange buffer (plain
//     stores, no atomics, no dependent L2 round trips in the apply phase);
//   * the same segment is written, with the same stores, into the exchange buffer of every
//     other GPU of the job over NVLink (peer pointers, Xq::base[]) — the exchange step of the
//     multi-GPU merge loop is fused into the kernel, there is no NCCL call per merge;
//   * every block drains ALL segments of ALL GPUs, keeps the entries whose key it owns and
//     applies them to its partition; every GPU holds the full table, so every GPU elects the
//     same pair without a second exchange;
//   * the pair of a merge is elected WITHOUT an exchange: every block keeps an identical copy of the leading pairs
//     (the "front", exact counts, shared memory) and maintains it from the entries it drains anyway; the front is
//     rebuilt from the partitions every few hundred merges (see "the replicated FRONT" below);
//   * a block parks the drained entries it owns in shared memory and adds them to its partition while it waits for
//     the other blocks' next count words, so the table's L2 round trips are off the critical path of a merge.
// There is NO grid barrier in the loop and ONE store -> load hop per merge: a block ends its apply phase by storing
// "round | flags | entries" for its segment; a block starts its drain by polling those words of all blocks (of all
// GPUs) until they carry the round — barrier and count fetch are one round trip; the entries carry their own stamps
// (no fence).  Tried before and slower: two cg grid.sync() + separate fetches; stamped words with every block polling
// every block's best (the sector requests of a poll round queue at a few L2 slices); a last-arriver / block-0 reducer
// (two more hops and the skew of the owner's partition sweep).
// The launch is still cooperative: all blocks must be co-resident for the polling to terminate.
// Words live in TILES: RESIDENT mode keeps tile b in the shared memory of block b for the whole
// launch; STREAMING mode (token buffer larger than the chip's shared memory) stages tiles through
// a TMA ring every merge (see below).
#pragma once

constexpr int SWEEP_UNROLL = 8;  // partition sweep: table counts in flight per thread

// ---- exchange buffer ("xq") --------------------------------------------------------------------
// Every rank owns one region: [parity 0/1][sender 0..world-1]{ XqHdr, entries[nblocks][seg_cap] }.
// Round r (r = 1, 2, ...) uses parity r & 1.  Block b of sender s writes its entries into segment
// [r & 1][s][b] of EVERY rank's region (its own included) and then the count word of that segment:
// (r << 32) | flags | entries.  Double buffering suffices: a block writes round r + 2 only after it has
// seen every block's count word of round r + 1 (it drains round r + 1 before it can elect the next pair),
// and a block stores that word after its apply phase r + 1, i.e. after it has finished draining round r.
constexpr int XQ_MAX_WORLD = 8;
constexpr int XQ_MAX_BLOCKS = 256;
constexpr uint32_t XQF_COMPACT = 1u;     // some block wants a compaction of its packed words
constexpr uint32_t XQF_OVERFLOW = 2u;    // a segment overflowed: counts are stale, rebuild the table
constexpr uint32_t XQF_MORE = 4u;        // out-of-loop table rounds: a sender has more chunks to publish
constexpr uint32_t XQF_PLIMIT = 8u;      // a partition is over the load limit: rebuild (dead keys vanish)
constexpr uint32_t XQF_PFULL = 16u;      // a partition ran full: grow the table
constexpr uint32_t XQ_CNT_OVF = 0x80000000u;      // count word: the segment overflowed
constexpr uint32_t XQ_CNT_MORE = 0x40000000u;     // count word (table rounds): further entries follow in the next round
constexpr uint32_t XQ_CNT_COMPACT = 0x20000000u;  // count word: > 25 % of the block's token slots are dead
constexpr uint32_t XQ_CNT_PLIMIT = 0x10000000u;   // count word: the block's partition is over the load limit
constexpr uint32_t XQ_CNT_PFULL = 0x08000000u;    // count word: the block's partition ran full (an update was lost)
constexpr uint32_t XQ_CNT_MASK = 0x07ffffffu;
// ORs the XQF_* flags of count word c into `flags`.  XQ_CNT_MORE is only set by the out-of-loop table rounds: `more`
// says whether to map it.
__device__ __forceinline__ void cnt_flags(uint32_t &flags, uint32_t c, bool more) {
  if (c & XQ_CNT_OVF) flags |= XQF_OVERFLOW;
  if (more && (c & XQ_CNT_MORE)) flags |= XQF_MORE;
  if (c & XQ_CNT_COMPACT) flags |= XQF_COMPACT;
  if (c & XQ_CNT_PLIMIT) flags |= XQF_PLIMIT;
  if (c & XQ_CNT_PFULL) flags |= XQF_PFULL;
}
// What bounds the exchange is the SM's load/store unit, not L2: a warp-wide load or store costs ~2 cycles per
// 128-byte line it touches, so 32 lanes on 32 lines are 64 cycles, and a POLL LOOP that does this from 16 warps keeps
// the unit busy for a microsecond per sweep.  Hence the layout:
//   * count words: one ROW per reader block (XqHdr::counts[reader][sender]) — the words a block polls are consecutive
//     (a warp's poll touches 2 lines) and are read by nobody else (no hot L2 lines);
//   * the first XQ_BOX entries of every segment sit in a place-major MATRIX (XqHdr::places[place][sender]): lanes that
//     handle the same place of consecutive senders read consecutive 16-byte slots (4 lines per warp);
//   * entries XQ_BOX.. of a segment (the first rounds of a run) stay in the sender's own segment.
constexpr int XQ_BOX = 7;
struct XqHdr {
  // ROWS: the count word (round << 32) | flags | entries of the sender's segment b exists once per local READER block r, at
  // counts[r * XQ_MAX_BLOCKS + b]: the sender stores it nblocks times (posted stores to distinct lines), reader r polls
  // its own row — nblocks consecutive words that nobody else reads.  (With one word per segment, polled by every
  // block, a poll round was tens of thousands of sector requests on lines shared by every SM.)
  unsigned long long counts[XQ_MAX_BLOCKS * XQ_MAX_BLOCKS];
  uint4 places[XQ_BOX * XQ_MAX_BLOCKS];   // entry e (< XQ_BOX) of the sender's block b: places[e * XQ_MAX_BLOCKS + b]
  // count words of the merge loop for the readers of ANOTHER rank: one per sender block, polled by all blocks of that
  // rank.  (Per-reader rows across NVLink were 1036 eight-byte stores per block and merge at 8 GPUs: ~11 us of a 35 us
  // merge on the wire.  The rows above stay for the local readers and for the out-of-loop table rounds.)
  unsigned long long shared[XQ_MAX_BLOCKS];
};
// count word of sender block `sb` in the row of reader block `rb`
__device__ __forceinline__ unsigned long long *xq_cnt(XqHdr *h, uint32_t rb, uint32_t sb) { return &h->counts[(size_t)rb * XQ_MAX_BLOCKS + sb]; }
struct Xq {
  unsigned char *base[XQ_MAX_WORLD];  // region of every rank; base[me] is local memory
  uint32_t world, me, nblocks, seg_cap;
  unsigned long long per_sender;      // bytes of one {header, entries} slot
};
__device__ __forceinline__ unsigned char *xq_base(const Xq &x, uint32_t rank) {
  unsigned char *p = x.base[0];
#pragma unroll
  for (int d = 1; d < XQ_MAX_WORLD; d++)
    if ((uint32_t)d == rank) p = x.base[d];
  return p;
}
__device__ __forceinline__ XqHdr *xq_hdr(const Xq &x, uint32_t rank, uint32_t parity, uint32_t sender) {
  return reinterpret_cast<XqHdr *>(xq_base(x, rank) + (size_t)(parity * x.world + sender) * x.per_sender);
}
// byte offset (inside any rank's region) of segment `block` of (parity, sender)
__device__ __forceinline__ size_t xq_seg_off(const Xq &x, uint32_t parity, uint32_t sender, uint32_t block) {
  return (size_t)(parity * x.world + sender) * x.per_sender + sizeof(XqHdr) + (size_t)block * x.seg_cap * sizeof(uint4);
}
// release store / acquire load of a stamped word in (possibly peer) global memory; sys: system scope (NVLink peers)
__device__ __forceinline__ void st_release(unsigned long long *p, unsigned long long v, bool sys) {
#ifndef YT_SIMT_EMU
  if (sys) asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
  else asm volatile("st.release.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
#else
  __atomic_store_n(p, v, __ATOMIC_RELEASE);
#endif
}
__device__ __forceinline__ unsigned long long ld_acquire(const unsigned long long *p, bool sys) {
#ifndef YT_SIMT_EMU
  unsigned long long v;
  if (sys) asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  else asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
#else
  return __atomic_load_n(p, __ATOMIC_ACQUIRE);
#endif
}
__device__ __forceinline__ unsigned long long ld_relaxed(const unsigned long long *p) {
#ifndef YT_SIMT_EMU
  unsigned long long v;
  asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
#else
  return __atomic_load_n(p, __ATOMIC_RELAXED);
#endif
}
__device__ __forceinline__ unsigned long long ld_relaxed_any(const unsigned long long *p, bool sys) {
#ifndef YT_SIMT_EMU
  unsigned long long v;
  if (sys) asm volatile("ld.relaxed.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  else asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
#else
  return __atomic_load_n(p, __ATOMIC_RELAXED);
#endif
}
// two consecutive 64-bit words (16-byte aligned) with one relaxed load
__device__ __forceinline__ void ld_relaxed2(const unsigned long long *p, unsigned long long *a, unsigned long long *b, bool sys) {
#ifndef YT_SIMT_EMU
  if (sys) asm volatile("ld.relaxed.sys.global.v2.u64 {%0, %1}, [%2];" : "=l"(*a), "=l"(*b) : "l"(p) : "memory");
  else asm volatile("ld.relaxed.gpu.global.v2.u64 {%0, %1}, [%2];" : "=l"(*a), "=l"(*b) : "l"(p) : "memory");
#else
  *a = __atomic_load_n(p, __ATOMIC_RELAXED);
  *b = __atomic_load_n(p + 1, __ATOMIC_RELAXED);
#endif
}
__device__ __forceinline__ void st_relaxed_any(unsigned long long *p, unsigned long long v, bool sys) {
#ifndef YT_SIMT_EMU
  if (sys) asm volatile("st.relaxed.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
  else asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
#else
  __atomic_store_n(p, v, __ATOMIC_RELAXED);
#endif
}
__device__ __forceinline__ void st_relaxed(unsigned long long *p, unsigned long long v) {
#ifndef YT_SIMT_EMU
  asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
#else
  __atomic_store_n(p, v, __ATOMIC_RELAXED);
#endif
}

// Token ids must fit 22 bits (the packed exchange entries below).
constexpr uint32_t BB_ID_LIMIT = 1u << 22;

// Exchange ENTRIES are self-stamped too (the scheme of NCCL's LL protocol): an entry is two 64-bit words, each carrying
// the low bits of its round, so neither the producer needs a fence between its entries and its count word nor the
// consumer an acquire — an entry whose stamps are not the round's has simply not arrived yet (NVLink and L2 deliver an
// aligned 8-byte word whole; nothing orders different addresses without a fence, and a system-scope fence after peer
// stores cost microseconds per merge).  w0 = stamp20 | x22 | y22, w1 = stamp20 | value44 (signed).
// stamp = round % 0xfffff, never 0xfffff: the buffer starts as all-ones.  (The round counter runs on across the runs and
// the kept trainings of a context, so stamps do repeat: a slot left untouched for exactly k * 0xfffff rounds of its parity
// carries a matching stamp again, and is then read wrongly only in the few hundred nanoseconds before its new content lands.)
constexpr uint32_t XQ_STAMP_MOD = 0xfffffu;
__device__ __forceinline__ uint4 xq_pack(uint32_t stamp, unsigned long long key, long long value) {
  const unsigned long long st = (unsigned long long)stamp << 44;
  const unsigned long long w0 = st | ((key >> 32) << 22) | (key & 0x3fffffull);
  const unsigned long long w1 = st | ((unsigned long long)value & 0xfffffffffffull);
  return make_uint4((uint32_t)w0, (uint32_t)(w0 >> 32), (uint32_t)w1, (uint32_t)(w1 >> 32));
}
// true when both words carry `stamp`; then *key / *value hold the entry
__device__ __forceinline__ bool xq_unpack(unsigned long long w0, unsigned long long w1, uint32_t stamp, unsigned long long *key,
                                          long long *value) {
  if ((uint32_t)(w0 >> 44) != stamp || (uint32_t)(w1 >> 44) != stamp) return false;
  *key = (((w0 >> 22) & 0x3fffffull) << 32) | (w0 & 0x3fffffull);
  *value = (long long)(w1 << 20) >> 20;   // sign-extend 44 bits
  return true;
}

struct LoopArgs {
  uint32_t *tok;
  const uint32_t *off;
  const uint64_t *freq;
  uint64_t n_words;
  const uint2 *tile_desc;      // n_tiles + 1 entries (first word, its token offset); last = (n_words, n_slots)
  uint32_t stream_tok_cap;     // STREAMING: token / word capacity of ONE pipeline stage
  uint32_t stream_word_cap;
  uint32_t n_stage;            // STREAMING: pipeline depth
  uint4 *defer;                // STREAMING: per-block lists of words to rewrite after the tile scan
  uint32_t defer_cap;          // entries per block
  uint32_t n_tiles;
  uint32_t resident;           // 1: block b owns tile b and keeps it in shared memory
  uint32_t smem_tok_cap;       // token capacity of the shared tile buffer
  uint32_t smem_word_cap;      // word capacity of the shared tile buffer
  PairTab tab;                 // tab.nparts == gridDim.x
  Xq xq;
  YtLoopCtl *ctl;
  unsigned long long *frontbuf;   // gather buffer of the front refreshes (front_buf_words()); cleared before every launch
  uint32_t *rules;                // 3 per merge
  unsigned long long *rfreq;
  uint32_t first_new_id;          // id of merge number 0
  uint32_t max_total;             // stop when ctl->n_done reaches this
  uint32_t max_iters;             // iterations allowed in this launch
  uint32_t part_limit;            // leave for a rebuild when a partition holds more keys than this
  uint32_t dead_min_slots;        // a block wishes a compaction only if it owns more token slots than this
  unsigned long long spin_limit_ns;  // a peer that stays silent this long traps the kernel (never hang the box)
  uint32_t front_top;                // pairs a partition contributes to a front refresh (1 .. FRONT_TOP)
  uint32_t newp_limit;               // keys the new-pair table takes per round (NEWP_LIMIT; tests: YTTM_NEWP_LIMIT)
  uint32_t drain_places;             // places per segment the drain covers with per-thread items (1 .. XQ_BOX); the rest of a
                                     // segment goes through the shared walk.  Host: as many as one trip of the items holds.
};

struct Best { unsigned long long c, prio, slot; };
__device__ __forceinline__ bool better(const Best &a, const Best &b) {  // a beats b
  return a.c > b.c || (a.c == b.c && a.prio > b.prio);
}
#ifndef YT_SIMT_EMU
__device__ __forceinline__ unsigned long long gtimer() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
  return t;
}
__device__ __forceinline__ void loop_trap() { asm volatile("trap;"); }
#else   // tests/emul/simt: the CPU clock
inline unsigned long long gtimer() {
  timespec ts;
  clock_gettime(CLOCK_MONOTONIC, &ts);
  return (unsigned long long)ts.tv_sec * 1000000000ull + (unsigned long long)ts.tv_nsec;
}
inline void loop_trap() { fprintf(stderr, "emu: merge loop gave up waiting for a peer\n"); abort(); }
#endif
// One trip of a wait on a peer: a peer that stays silent for limit_ns traps the kernel (never hang the box).  The clock
// is read every 4096 trips only; t0 = 0 before the first reading.  The emulator yields to the other fibers.
__device__ __forceinline__ void spin_step(uint32_t spin, unsigned long long &t0, unsigned long long limit_ns) {
#ifdef YT_SIMT_EMU
  emu::yield();
#endif
  if ((spin & 4095u) == 4095u) {
    if (!t0) t0 = gtimer();
    else if (gtimer() - t0 > limit_ns) loop_trap();
  }
}
__device__ __forceinline__ Best warp_best(Best v) {
  for (int o = 16; o > 0; o >>= 1) {
    Best w;
    w.c = __shfl_xor_sync(0xffffffffu, v.c, o);
    w.prio = __shfl_xor_sync(0xffffffffu, v.prio, o);
    w.slot = __shfl_xor_sync(0xffffffffu, v.slot, o);
    if (better(w, v)) v = w;
  }
  return v;
}

struct MergeOp { uint32_t x, y, z; unsigned long long key; };

constexpr int MAX_STAGES = 16;
constexpr int CLAIM_WORDS = 1024;  // claim bitmap: up to 32768 words per shared-memory tile

// This block's outgoing segment of the current round: the same offset in every rank's region.
struct XqOut {
  size_t off;        // byte offset of the segment inside a region
  uint32_t *s_n;     // shared-memory entry counter of the block (may run past cap: overflow)
  uint32_t stamp;    // round % XQ_STAMP_MOD of the entries
  uint32_t parity;   // round & 1
};
__device__ __forceinline__ void xq_store(const LoopArgs &a, const XqOut &o, uint32_t i, unsigned long long key,
                                         long long delta) {
  if (i >= a.xq.seg_cap) return;  // overflow: the count word carries the flag, the host rebuilds the table
  const uint4 e = xq_pack(o.stamp, key, delta);
  if (i < (uint32_t)XQ_BOX) {   // the place-major matrix of the round
#pragma unroll
    for (int d = 0; d < XQ_MAX_WORLD; d++)
      if ((uint32_t)d < a.xq.world) xq_hdr(a.xq, (uint32_t)d, o.parity, a.xq.me)->places[i * XQ_MAX_BLOCKS + blockIdx.x] = e;
    return;
  }
#pragma unroll
  for (int d = 0; d < XQ_MAX_WORLD; d++)
    if ((uint32_t)d < a.xq.world) reinterpret_cast<uint4 *>(a.xq.base[d] + o.off)[i] = e;
}
// one thread on its own (scalar paths)
__device__ __forceinline__ void xq_push1(const LoopArgs &a, const XqOut &o, unsigned long long key, long long delta) {
  xq_store(a, o, atomicAdd(o.s_n, 1u), key, delta);
}
// One thread rewrites word t (`cap` token slots) that holds (x,y): -old pairs, rewrite, +new pairs.  The merges are
// added to `merges` (a 32- or 64-bit counter).
template <class N>
__device__ __forceinline__ void apply_word_scalar(uint32_t *t, uint32_t cap, long long f, const MergeOp &op,
                                                  const LoopArgs &a, const XqOut &xo, N &merges) {
  for_each_pair(t, cap, [&](uint64_t key, uint64_t mult) {
    if (key != op.key) xq_push1(a, xo, key, -(long long)mult * f);
  });
  merges += rewrite_word(t, cap, op.x, op.y, op.z);
  for_each_pair(t, cap, [&](uint64_t key, uint64_t mult) { xq_push1(a, xo, key, (long long)mult * f); });
}

// Run structure of <= 32 live tokens held one per lane (t == DEAD beyond the n live ones): every
// run start owns floor(L/2) self pairs and one cross pair to the next run (for_each_pair()).
struct RunInfo { bool start; uint32_t nxt, L, b; unsigned starts; };
__device__ __forceinline__ RunInfo warp_runs(uint32_t t, uint32_t n, unsigned lane) {
  RunInfo r;
  const bool valid = lane < n;
  uint32_t prev = __shfl_up_sync(0xffffffffu, t, 1);
  r.start = valid && (lane == 0 || prev != t);
  r.starts = __ballot_sync(0xffffffffu, r.start);
  const unsigned above = lane == 31 ? 0u : r.starts & ~((2u << lane) - 1u);
  r.nxt = above ? (uint32_t)__ffs(above) - 1u : n;
  r.b = __shfl_sync(0xffffffffu, t, r.nxt & 31);
  r.L = r.nxt - lane;
  return r;
}

// One warp rewrites one word that holds (x,y): st = its `cap` token slots (shared or global
// memory), gt = optional write-through copy in global memory.  Count changes: only the pairs
// whose run is touched by a merge are emitted (-old, +new); untouched runs cancel exactly.
// Returns the number of merges.
__device__ __forceinline__ uint32_t warp_apply_word(uint32_t *st, uint32_t cap, uint32_t *gt, long long f,
                                                    const MergeOp &op, unsigned lane, const LoopArgs &a,
                                                    const XqOut &xo) {
  if (cap > 32) {  // long word: scalar path on lane 0 (exact, slow)
    uint32_t merges = 0;
    if (lane == 0) apply_word_scalar(st, cap, f, op, a, xo, merges);
    __syncwarp();
    if (gt)
      for (uint32_t i = lane; i < cap; i += 32) gt[i] = st[i];
    return __shfl_sync(0xffffffffu, merges, 0);
  }
  const uint32_t t = lane < cap ? st[lane] : DEAD;
  const bool valid = t != DEAD;
  const uint32_t n = __popc(__ballot_sync(0xffffffffu, valid));  // live tokens form a prefix
  const RunInfo ro = warp_runs(t, n, lane);
  // greedy left-to-right matches
  const uint32_t nx = __shfl_down_sync(0xffffffffu, t, 1);
  bool m = valid && lane + 1 < n && t == op.x && nx == op.y;
  if (op.x == op.y) {  // inside a run x^L only every second position starts a pair (bpe.cpp:654-690)
    const unsigned upto = ro.starts & (lane == 31 ? 0xffffffffu : ((2u << lane) - 1u));
    const uint32_t run_start = upto ? 31u - (uint32_t)__clz(upto) : 0u;
    m = m && (((lane - run_start) & 1u) == 0u);
  }
  const unsigned mm = __ballot_sync(0xffffffffu, m);
  const unsigned touched = mm | (mm << 1);                       // first and second token of every merged pair
  const bool keep = valid && !((mm << 1) >> lane & 1u);
  const unsigned km = __ballot_sync(0xffffffffu, keep);
  const uint32_t newpos = __popc(km & ((1u << lane) - 1u));
  const uint32_t n2 = __popc(km);
  const uint32_t nv = m ? op.z : t;
  // an old run [lane, nxt) (plus the first token of the next run) without a touched token is unchanged
  const unsigned span_mask = (ro.nxt >= 31 ? 0xffffffffu : ((2u << ro.nxt) - 1u)) & ~((1u << lane) - 1u);
  const bool old_changed = ro.start && (touched & span_mask) != 0u;
  const unsigned unchanged_starts = __ballot_sync(0xffffffffu, ro.start && !old_changed);
  __syncwarp();  // every lane holds its old token in a register before any slot is overwritten
  if (keep) { st[newpos] = nv; if (gt) gt[newpos] = nv; }
  if (valid && lane >= n2) { st[lane] = DEAD; if (gt) gt[lane] = DEAD; }
  // new lane p came from old lane src = (p+1)-th kept lane: fetch its token with a shuffle (st may be
  // global memory in the deferred path: no re-read through L1); its run is unchanged iff that old run was
  const uint32_t src = lane < n2 ? __fns(km, 0, lane + 1) : 0u;
  const uint32_t moved = __shfl_sync(0xffffffffu, nv, src & 31);
  const uint32_t t2 = lane < n2 ? moved : DEAD;
  const RunInfo rn = warp_runs(t2, n2, lane);
  const bool new_changed = rn.start && !((unchanged_starts >> (src & 31)) & 1u);
  // the four possible updates of this lane
  const bool h0 = old_changed && ro.L >= 2 && pair_key(t, t) != op.key;
  const bool h1 = old_changed && ro.nxt < n && pair_key(t, ro.b) != op.key;
  const bool h2 = new_changed && rn.L >= 2;
  const bool h3 = new_changed && rn.nxt < n2;
  {  // one reservation in the segment for all four kinds (a returning shared-memory atomic costs ~100 cycles)
    const unsigned m0 = __ballot_sync(0xffffffffu, h0), m1 = __ballot_sync(0xffffffffu, h1);
    const unsigned m2 = __ballot_sync(0xffffffffu, h2), m3 = __ballot_sync(0xffffffffu, h3);
    const uint32_t c0 = __popc(m0), c1 = __popc(m1), c2 = __popc(m2), tot = c0 + c1 + c2 + __popc(m3);
    if (tot) {
      uint32_t base = 0;
      if (lane == 0) base = atomicAdd(xo.s_n, tot);
      base = __shfl_sync(0xffffffffu, base, 0);
      const unsigned below = (1u << lane) - 1u;
      if (h0) xq_store(a, xo, base + __popc(m0 & below), pair_key(t, t), -f * (long long)(ro.L >> 1));
      if (h1) xq_store(a, xo, base + c0 + __popc(m1 & below), pair_key(t, ro.b), -f);
      if (h2) xq_store(a, xo, base + c0 + c1 + __popc(m2 & below), pair_key(t2, t2), f * (long long)(rn.L >> 1));
      if (h3) xq_store(a, xo, base + c0 + c1 + c2 + __popc(m3 & below), pair_key(t2, rn.b), f);
    }
  }
  return n - n2;
}

// Bit k: token k and token k+1 of the eight tokens v, u, nxt are (x,y).
__device__ __forceinline__ uint32_t match8(const uint4 &v, const uint4 &u, uint32_t nxt, const MergeOp &op) {
  return (v.x == op.x && v.y == op.y ? 1u : 0u) | (v.y == op.x && v.z == op.y ? 2u : 0u) |
         (v.z == op.x && v.w == op.y ? 4u : 0u) | (v.w == op.x && u.x == op.y ? 8u : 0u) |
         (u.x == op.x && u.y == op.y ? 16u : 0u) | (u.y == op.x && u.z == op.y ? 32u : 0u) |
         (u.z == op.x && u.w == op.y ? 64u : 0u) | (u.w == op.x && nxt == op.y ? 128u : 0u);
}
// The word that holds token i: the largest w < nw with off[w] - base <= i.
__device__ __forceinline__ uint32_t word_at(const uint32_t *off, uint32_t nw, uint32_t i, uint32_t base) {
  uint32_t lo = 0, hi = nw;
  while (hi - lo > 1) {
    const uint32_t mid = (lo + hi) >> 1;
    if (off[mid] - base <= i) lo = mid; else hi = mid;
  }
  return lo;
}

// One RESIDENT tile: its token slots sit in shared memory (`span` slots at stok, word w at
// [soff[w], soff[w+1])).  The scan is TOKEN-parallel: a lane compares four consecutive slots and
// the one after them with (x, y) — consecutive lanes read consecutive 16-byte pieces of shared
// memory, every lane does the same work whatever the word lengths.  A hit cannot straddle two words: the first token
// of every word is (derived from) the "▁" token, which only ever occurs at position 0, so y —
// the second element of an in-word pair — is never a word-initial token; tail padding (DEAD)
// matches nothing.  Each hit is mapped to its word (binary search in the offsets), the word is
// claimed once through a bitmap, and claimed words are rewritten by the whole warp.
__device__ __forceinline__ unsigned long long process_tile(uint32_t *stok, const uint32_t *soff, uint32_t nw,
                                                           uint32_t span, uint32_t *claim, const uint64_t *gfreq,
                                                           const MergeOp &op, const LoopArgs &a, const XqOut &xo) {
  const unsigned lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nwarp = blockDim.x >> 5;
  unsigned long long dead = 0;
  // a lane compares eight tokens from two 16-byte shared loads (stok is 16-byte aligned, its capacity a multiple
  // of 4); the token after them comes from the next lane.  (Four per lane: twice the trips; the loop is latency bound —
  // one warp issues a dependent instruction every ~5 cycles — so instructions per token are what counts.)
  for (uint32_t base = wid * 256; base < span; base += nwarp * 256) {
    const uint32_t p = base + lane * 8;
    uint4 v = make_uint4(DEAD, DEAD, DEAD, DEAD), u = v;
    if (p < span) v = *reinterpret_cast<const uint4 *>(stok + p);
    if (p + 4 < span) u = *reinterpret_cast<const uint4 *>(stok + p + 4);
    uint32_t nxt = __shfl_down_sync(0xffffffffu, v.x, 1);
    if (lane == 31) nxt = p + 8 < span ? stok[p + 8] : DEAD;
    uint32_t m = match8(v, u, nxt, op);
    if (p + 8 >= span) m &= span > p + 1 ? (1u << (span - p - 1)) - 1u : 0u;  // occurrence i needs i + 1 < span
    while (__ballot_sync(0xffffffffu, m != 0)) {  // one round per hit of the busiest lane (almost always one)
      uint32_t w = 0, o = 0, cap = 0;
      bool own = false;
      if (m) {
        const uint32_t i = p + (uint32_t)__ffs(m) - 1u;
        m &= m - 1u;
        // re-read: an earlier round (or another warp) may already have rewritten this word
        if (stok[i] == op.x && stok[i + 1] == op.y) {
          w = word_at(soff, nw, i, 0);
          o = soff[w];
          cap = soff[w + 1] - o;
          own = !((atomicOr(&claim[w >> 5], 1u << (w & 31)) >> (w & 31)) & 1u);
        }
      }
      const long long fw = own ? (long long)gfreq[w] : 0;  // owners fetch their word's frequency together
      unsigned mask = __ballot_sync(0xffffffffu, own);
      while (mask) {
        const int j = __ffs(mask) - 1;
        mask &= mask - 1;
        const uint32_t oj = __shfl_sync(0xffffffffu, o, j), cj = __shfl_sync(0xffffffffu, cap, j);
        const uint32_t wj = __shfl_sync(0xffffffffu, w, j);
        const long long f = __shfl_sync(0xffffffffu, fw, j);
        dead += warp_apply_word(stok + oj, cj, nullptr, f, op, lane, a, xo);
        if (lane == 0) atomicAnd(&claim[wj >> 5], ~(1u << (wj & 31)));  // bitmap all zero between tiles
      }
    }
  }
  return lane == 0 ? dead : 0ull;
}

// Oversized tile (a word longer than the shared buffer): thread per word straight on global memory.
__device__ __forceinline__ unsigned long long process_tile_direct(uint32_t *tok, const uint32_t *off,
                                                                  const uint64_t *freq, uint32_t w0, uint32_t w1,
                                                                  const MergeOp &op, const LoopArgs &a, const XqOut &xo) {
  unsigned long long dead = 0;
  for (uint32_t w = w0 + threadIdx.x; w < w1; w += blockDim.x) {
    uint32_t o = off[w], wcap = off[w + 1] - o;
    uint32_t *t = tok + o;
    if (!has_pair(t, wcap, op.x, op.y)) continue;
    apply_word_scalar(t, wcap, (long long)freq[w], op, a, xo, dead);
  }
  return dead;
}

// ---- TMA (bulk async copy) staging of a tile: global -> shared, completion on an mbarrier ----------
#ifndef YT_SIMT_EMU
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long *bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(unsigned long long *bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_bulk_g2s(void *dst, const void *src, uint32_t bytes, unsigned long long *bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(dst)),
               "l"(src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(unsigned long long *bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long *bar, uint32_t parity) {
  uint32_t ok = 0;
  for (uint32_t spin = 0; !ok; spin++) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    if (spin > (1u << 28)) asm volatile("trap;");  // a lost transaction must not hang the box
  }
}
#else
// tests/emul/simt (CPU emulation of the kernels, test harness only): the mbarrier word is modelled as
// { pending arrivals : 16, arrival count : 16, outstanding transaction bytes : 31, phase : 1 }; a bulk copy is an
// immediate memcpy that completes its bytes on the barrier; a waiter yields to the other fibers of the block.
struct EmuMbar { uint64_t pending : 16, count : 16, tx : 31, phase : 1; };
inline EmuMbar *emu_bar(unsigned long long *bar) { return reinterpret_cast<EmuMbar *>(bar); }
inline void emu_bar_check(EmuMbar *m) {
  if (m->pending == 0 && m->tx == 0) { m->phase ^= 1u; m->pending = m->count; }
}
inline void mbar_init(unsigned long long *bar, uint32_t count) {
  EmuMbar *m = emu_bar(bar);
  m->pending = count; m->count = count; m->tx = 0; m->phase = 0;
}
inline void mbar_expect_tx(unsigned long long *bar, uint32_t bytes) {  // one arrival + expected bytes
  EmuMbar *m = emu_bar(bar);
  m->tx += bytes;
  m->pending -= 1;
  emu_bar_check(m);
}
inline void tma_bulk_g2s(void *dst, const void *src, uint32_t bytes, unsigned long long *bar) {
  if (((uintptr_t)dst | (uintptr_t)src | bytes) & 15u) { fprintf(stderr, "emu: misaligned bulk copy\n"); abort(); }
  memcpy(dst, src, bytes);
  EmuMbar *m = emu_bar(bar);
  m->tx -= bytes;
  emu_bar_check(m);
}
inline void mbar_arrive(unsigned long long *bar) {
  EmuMbar *m = emu_bar(bar);
  m->pending -= 1;
  emu_bar_check(m);
}
inline void mbar_wait(unsigned long long *bar, uint32_t parity) {  // returns once the phase of that parity is over
  for (uint64_t spin = 0; emu_bar(bar)->phase == (parity & 1u); spin++) {
    if (spin > (1u << 24)) { fprintf(stderr, "emu: mbarrier wait never completes\n"); abort(); }
    emu::yield();
  }
}
#endif
// Tile descriptors travel in lane-distributed batches: lane j of a warp holds tile_desc[base + j], and tile base + j
// (j < 31) takes its first and last descriptor (d0, d1) from lanes j and j + 1.
__device__ __forceinline__ void tile_pair(uint2 batch, uint32_t j, uint2 &d0, uint2 &d1) {
  d0.x = __shfl_sync(0xffffffffu, batch.x, j);     d0.y = __shfl_sync(0xffffffffu, batch.y, j);
  d1.x = __shfl_sync(0xffffffffu, batch.x, j + 1); d1.y = __shfl_sync(0xffffffffu, batch.y, j + 1);
}
// bytes of a 16-byte aligned window [lo & ~3, roundup(hi, 4)) over uint32 elements
__device__ __forceinline__ uint32_t win_lo(uint32_t lo) { return lo & ~3u; }
__device__ __forceinline__ uint32_t win_bytes(uint32_t lo, uint32_t hi) { return (((hi + 3u) & ~3u) - (lo & ~3u)) * 4u; }

__device__ __forceinline__ void load_tile(const LoopArgs &a, uint32_t w0, uint32_t w1, uint32_t *stok, uint32_t *soff) {
  const uint32_t o0 = a.off[w0], span = a.off[w1] - o0, nw = w1 - w0;  // resident mode: plain coalesced copy, once
  for (uint32_t i = threadIdx.x; i <= nw; i += blockDim.x) soff[i] = a.off[w0 + i] - o0;
  const uint32_t *src = a.tok + o0;
  for (uint32_t i = threadIdx.x; i < span; i += blockDim.x) stok[i] = __ldcg(src + i);
}

#ifndef YT_SIMT_EMU
extern __shared__ __align__(16) uint32_t yt_dyn_smem[];
#else
#define yt_dyn_smem (reinterpret_cast<uint32_t *>(emu::dyn_smem()))
#endif

// Poll the count words of round `round` of every (sender, block) segment in this rank's region until they carry the
// round, and leave the entry counts in s_pref[0 .. world * nblocks).  Barrier and count fetch in one: a word becomes
// visible after its block's entries (release / acquire).  Thread t owns the consecutive segments [t * ipt, (t+1) * ipt).
// Returns (block-uniform, through *s_acc) the OR of XQF_* flags seen; skip_self: this rank's own segments count as empty.
__device__ __forceinline__ void xq_poll_counts(const LoopArgs &a, uint32_t round, bool skip_self, uint32_t *s_pref,
                                               uint32_t *s_acc) {
  const uint32_t nseg = a.xq.world * a.xq.nblocks, parity = round & 1u;
  const uint32_t ipt = (nseg + blockDim.x - 1) / blockDim.x;
  const bool sys = a.xq.world > 1;
  uint32_t flags = 0;
  unsigned long long t0 = 0;
  for (uint32_t k = 0; k < ipt; k++) {
    const uint32_t j = threadIdx.x * ipt + k;
    if (j >= nseg) break;
    const uint32_t s = j / a.xq.nblocks, b = j - s * a.xq.nblocks;
    const unsigned long long *w = xq_cnt(xq_hdr(a.xq, a.xq.me, parity, s), blockIdx.x, b);
    unsigned long long v;
    for (uint32_t spin = 0;; spin++) {
      v = ld_relaxed_any(w, sys);   // entries validate themselves: no acquire needed
      if ((uint32_t)(v >> 32) == round) break;
      spin_step(spin, t0, a.spin_limit_ns);
    }
    const uint32_t c = (uint32_t)v;
    cnt_flags(flags, c, true);
    uint32_t n = c & XQ_CNT_MASK;
    if (n > a.xq.seg_cap) n = a.xq.seg_cap;
    s_pref[j] = (skip_self && s == a.xq.me) ? 0u : n;
  }
  if (flags) atomicOr(s_acc, flags);
  __syncthreads();
}

// Drain of the out-of-loop table rounds (xq_absorb_kernel): s_pref holds the entry counts (xq_poll_counts); every entry
// whose key belongs to partition blockIdx.x is added to that partition.  *s_occ_add is increased by the keys inserted.
__device__ __forceinline__ void xq_prefix(const LoopArgs &a, uint32_t *s_pref, uint32_t *s_scan /* 33 words */) {
  const unsigned lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nwarp = blockDim.x >> 5;
  const uint32_t nseg = a.xq.world * a.xq.nblocks;
  const uint32_t ipt = (nseg + blockDim.x - 1) / blockDim.x;
  // ---- exclusive prefix of the segment sizes, in place; s_pref[nseg] = total
  uint32_t mine = 0;
  for (uint32_t k = 0; k < ipt; k++) {
    const uint32_t j = threadIdx.x * ipt + k;
    if (j < nseg) mine += s_pref[j];
  }
  uint32_t x = mine;
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= (unsigned)o) x += y;
  }
  if (lane == 31) s_scan[wid] = x;
  __syncthreads();
  if (wid == 0) {
    const uint32_t v = lane < nwarp ? s_scan[lane] : 0u;
    uint32_t xs = v;
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t y = __shfl_up_sync(0xffffffffu, xs, o);
      if (lane >= (unsigned)o) xs += y;
    }
    s_scan[lane] = xs - v;
    if (lane == 31) s_scan[32] = xs;
  }
  __syncthreads();
  {
    uint32_t run = s_scan[wid] + x - mine;  // exclusive prefix of this thread's first item
    for (uint32_t k = 0; k < ipt; k++) {
      const uint32_t j = threadIdx.x * ipt + k;
      if (j < nseg) { const uint32_t c = s_pref[j]; s_pref[j] = run; run += c; }
    }
  }
  if (threadIdx.x == 0) s_pref[nseg] = s_scan[32];
  __syncthreads();
}
// entry i (0 <= i < s_pref[nseg]) of round `round` in this rank's region; spins until both words carry the round's stamp
// first: number of the first entry this walk covers (the merge loop: the entries its per-place items left over)
__device__ __forceinline__ void xq_entry(const LoopArgs &a, uint32_t round, const uint32_t *s_pref, uint32_t i,
                                         unsigned long long *key, long long *delta, uint32_t first = 0) {
  const uint32_t nseg = a.xq.world * a.xq.nblocks;
  uint32_t lo = 0, hi = nseg;  // largest j with s_pref[j] <= i (empty segments share a prefix value: take the last)
  while (hi - lo > 1) {
    const uint32_t mid = (lo + hi) >> 1;
    if (s_pref[mid] <= i) lo = mid; else hi = mid;
  }
  const uint32_t s = lo / a.xq.nblocks, b = lo - s * a.xq.nblocks;
  const uint32_t idx = i - s_pref[lo] + first;   // the entry's number inside its segment
  const unsigned long long *ep = first && idx < (uint32_t)XQ_BOX   // (the merge loop: entries 0 .. XQ_BOX-1 sit in the place matrix)
      ? reinterpret_cast<const unsigned long long *>(xq_hdr(a.xq, a.xq.me, round & 1u, s)->places + idx * XQ_MAX_BLOCKS + b)
      : reinterpret_cast<const unsigned long long *>(xq_base(a.xq, a.xq.me) + xq_seg_off(a.xq, round & 1u, s, b) + (size_t)idx * sizeof(uint4));
  const bool sys = a.xq.world > 1;
  unsigned long long t0 = 0;
  for (uint32_t spin = 0; !xq_unpack(ld_relaxed_any(ep, sys), ld_relaxed_any(ep + 1, sys), round % XQ_STAMP_MOD, key, delta); spin++)
    spin_step(spin, t0, a.spin_limit_ns);   // the count word overtook the entry: it is on its way
}
__device__ __forceinline__ void xq_drain(const LoopArgs &a, uint32_t round, uint32_t *s_pref, uint32_t *s_scan /* 33 words */,
                                         uint32_t *s_occ_add) {
  xq_prefix(a, s_pref, s_scan);
  const uint32_t nseg = a.xq.world * a.xq.nblocks, total = s_pref[nseg];
  const uint32_t R = a.tab.rmask + 1;
  uint32_t added = 0;
  for (uint32_t i = threadIdx.x; i < total; i += blockDim.x) {
    unsigned long long key = 0;
    long long delta = 0;
    xq_entry(a, round, s_pref, i, &key, &delta);
    const uint64_t hh = mix64(key);
    if (pair_part(a.tab, hh) != blockIdx.x) continue;
    added += pair_add_at(a.tab, (uint64_t)blockIdx.x * R, (uint32_t)hh & a.tab.rmask, key, delta) ? 1u : 0u;
  }
  if (added) atomicAdd(s_occ_add, added);
}

// ---- the replicated FRONT ----------------------------------------------------------------------------------------
// Every block (of every GPU) keeps the same small set of leading pairs with their exact counts in shared memory and
// elects the pair of a merge from it, alone: every block reads every count change of a merge anyway (the drain), so the
// copies stay identical without a word being exchanged.  What makes this exact:
//   * pairs are totally ordered by (count, priority) — MergeCandidate::operator<, bpe.cpp:110-126;
//   * a REFRESH takes the FRONT_TOP leading pairs of every partition (its owner sweeps it, the blocks of a GPU gather
//     the lists through a small buffer) and sets BOUND = the largest FRONT_TOP-th pair of any partition: every pair
//     above the bound is in the front;
//   * the count of a pair outside the front can only fall (a merge only removes occurrences of existing tokens), except
//     for the pairs of the token created by the merge itself: those are aggregated per round and enter the front if
//     they are not below the bound.  Hence "every pair outside the front is below the bound" holds between refreshes,
//     and the largest member of the front is the global arg-max as long as it is not below the bound;
//   * otherwise (front exhausted, front too full, too many new pairs in one round) all blocks — they see the same
//     front — refresh in the same iteration.  A refresh costs FRONT_TOP partition sweeps and one gather, and pays for
//     a few hundred merges (one partition per SM x 8 pairs; the bound sits where the first partition runs out).
// The pair table in HBM/L2 stays the ground truth (rebuilds, refreshes, the multi-GPU table build): a block parks the
// entries it owns in shared memory during the drain and adds them to its partition while it waits for the other blocks'
// next count words — off the critical path of the merge.
// (Load factor: the drain looks every entry of a round up, mostly keys that are NOT in the front, and a miss walks to the
// end of its cluster; at 2048 slots / up to 1280 members the longest clusters of linear probing cost ~3 us per merge
// — some lane of some warp hit one every round.  4096 slots / <= 1024 members: clusters of a few slots.)
constexpr uint32_t FRONT_SLOTS = 4096;   // shared-memory hash table (key, count), per block
constexpr uint32_t FRONT_FILL = 1024;    // members that trigger a refresh (dead members are only dropped there)
constexpr uint32_t FRONT_LIST = FRONT_FILL + 1024 + 64;   // member list: a round adds at most NEWP_SLOTS members
constexpr uint32_t NEWP_SLOTS = 1024;    // the round's pairs with the new token, aggregated before they meet the bound
constexpr uint32_t NEWP_LIMIT = 768;     // keys the table takes; a round with more new pairs only BOUNDS them (sketch)
constexpr uint32_t NEWP_SKETCH = 1024;   // u64 buckets: sum of the counts of ALL new pairs of the round, by hash
constexpr uint32_t OWN_CAP = 256;        // parked entries of one round (more: added to the partition at once)
constexpr int FRONT_TOP = 6;             // most pairs a partition contributes to a refresh (LoopArgs::front_top, default 4)
constexpr int DRAIN_ITEMS = 3;           // (place, segment) items per thread and trip of the drain
constexpr size_t LOOP_FRONT_BYTES = ((size_t)FRONT_SLOTS * 2 + NEWP_SLOTS * 2 + OWN_CAP * 2) * 8 + ((size_t)NEWP_SLOTS + FRONT_LIST) * 4 + (size_t)NEWP_SKETCH * 8;
// global gather buffer of a refresh: [nblocks flag words, 128 bytes apart][nblocks x FRONT_TOP x (count, key)]
YT_HD size_t front_buf_words(uint32_t nblocks) { return (size_t)nblocks * 16 + (size_t)nblocks * FRONT_TOP * 2; }

__device__ __forceinline__ uint32_t smem_home(uint64_t hh, uint32_t mask) { return (uint32_t)(hh >> 20) & mask; }
// slot of `key` or ~0u (no insert may run concurrently)
__device__ __forceinline__ uint32_t smem_tab_find(const unsigned long long *keys, uint32_t mask, uint64_t hh, unsigned long long key) {
  uint32_t i = smem_home(hh, mask);
  for (uint32_t p = 0; p <= mask; p++, i = (i + 1) & mask) {
    const unsigned long long k = keys[i];
    if (k == key) return i;
    if (k == PK_EMPTY) return ~0u;
  }
  return ~0u;
}
// 64-bit add in shared memory out of two NATIVE 32-bit atomics (low word, then high word + carry).  atomicAdd on a
// 64-bit shared word compiles to a compare-and-swap loop (ATOMS.CAST.SPIN), and the count changes of a merge pile up
// on few keys (the new token next to its most frequent neighbours), where a loop retries.  (Introduced when the drain
// was thought to be atomics bound; the session that added it measured no gain by itself — the real limit was the
// load/store unit — it stayed because it bounds the work per add.)  The sum is exact
// once all adds have landed (nobody reads a count inside the drain).
__device__ __forceinline__ void smem_add64(unsigned long long *p, unsigned long long delta) {
  uint32_t *w = reinterpret_cast<uint32_t *>(p);   // little endian: w[0] low, w[1] high
  const uint32_t dlo = (uint32_t)delta, dhi = (uint32_t)(delta >> 32);
  uint32_t carry = 0;
  if (dlo) {
    const uint32_t old = atomicAdd(w, dlo);
    carry = old + dlo < old ? 1u : 0u;
  }
  if (dhi + carry) atomicAdd(w + 1, dhi + carry);
}
// insert-or-add; false: the table is full.  list (optional): the slots taken, in order of arrival (mask + 1 places)
__device__ __forceinline__ bool smem_tab_add(unsigned long long *keys, unsigned long long *cnts, uint32_t mask, uint64_t hh,
                                             unsigned long long key, long long delta, uint32_t *occ, uint32_t *list = nullptr) {
  uint32_t i = smem_home(hh, mask);
  for (uint32_t p = 0; p <= mask; p++, i = (i + 1) & mask) {
    unsigned long long k = *reinterpret_cast<volatile unsigned long long *>(keys + i);
    if (k == PK_EMPTY) {
      k = atomicCAS(keys + i, PK_EMPTY, key);
      if (k == PK_EMPTY) {
        const uint32_t q = atomicAdd(occ, 1u);
        if (list) list[q] = i;
        k = key;
      }
    }
    if (k == key) { smem_add64(cnts + i, (unsigned long long)delta); return true; }
  }
  return false;
}
// slot of `key`, inserted if absent; ~0u: absent and the table already holds `limit` keys
__device__ __forceinline__ uint32_t smem_tab_slot(unsigned long long *keys, uint32_t mask, uint64_t hh, unsigned long long key,
                                                  uint32_t *occ, uint32_t *list, uint32_t limit) {
  uint32_t i = smem_home(hh, mask);
  for (uint32_t p = 0; p <= mask; p++, i = (i + 1) & mask) {
    unsigned long long k = *reinterpret_cast<volatile unsigned long long *>(keys + i);
    if (k == PK_EMPTY) {
      if (*reinterpret_cast<volatile uint32_t *>(occ) >= limit) return ~0u;
      k = atomicCAS(keys + i, PK_EMPTY, key);
      if (k == PK_EMPTY) {
        const uint32_t q = atomicAdd(occ, 1u);
        if (list) list[q] = i;
        return i;
      }
    }
    if (k == key) return i;
  }
  return ~0u;
}
__device__ __forceinline__ unsigned long long prio_key(unsigned long long prio) {   // inverse of pair_prio
  const uint32_t mx = 0xffffffffu - (uint32_t)(prio >> 32), mn = 0x7fffffffu - (uint32_t)((prio & 0xffffffffull) >> 1);
  return (prio & 1ull) ? pair_key(mx, mn) : pair_key(mn, mx);
}
__device__ __forceinline__ void block_best(Best b, Best *s_warp, Best *s_out) {   // ends with a block barrier
  const unsigned lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nwarp = blockDim.x >> 5;
  b = warp_best(b);
  if (lane == 0) s_warp[wid] = b;
  __syncthreads();
  if (wid == 0) {
    Best v = lane < nwarp ? s_warp[lane] : Best{0, 0, 0};
    v = warp_best(v);
    if (lane == 0) *s_out = v;
  }
  __syncthreads();
}
// Warp arg-max of (count, priority) with four redux.sync instead of thirty shuffles; .slot must fit 32 bits.
__device__ __forceinline__ Best warp_best_redux(Best v) {
  const unsigned full = 0xffffffffu;
  bool ok = true;
  uint32_t m = __reduce_max_sync(full, (uint32_t)(v.c >> 32));
  ok = (uint32_t)(v.c >> 32) == m;
  uint32_t m2 = __reduce_max_sync(full, ok ? (uint32_t)v.c : 0u);
  ok = ok && (uint32_t)v.c == m2;
  const unsigned long long c = ((unsigned long long)m << 32) | m2;
  m = __reduce_max_sync(full, ok ? (uint32_t)(v.prio >> 32) : 0u);
  ok = ok && (uint32_t)(v.prio >> 32) == m;
  m2 = __reduce_max_sync(full, ok ? (uint32_t)v.prio : 0u);
  ok = ok && (uint32_t)v.prio == m2;
  const unsigned who = __ballot_sync(full, ok);   // never empty: the lanes that hold the maximum
  const uint32_t slot = __shfl_sync(full, (uint32_t)v.slot, __ffs(who) - 1);
  return Best{c, c ? ((unsigned long long)m << 32) | m2 : 0ull, slot};
}
// Block arg-max with ONE barrier: every warp reduces the per-warp results again, every thread returns the result.
// s_warp must not be written again before another block barrier.
__device__ __forceinline__ Best block_best_all(Best b, Best *s_warp) {
  const unsigned lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nwarp = blockDim.x >> 5;
  b = warp_best_redux(b);
  if (lane == 0) s_warp[wid] = b;
  __syncthreads();
  return warp_best_redux(lane < nwarp ? s_warp[lane] : Best{0, 0, 0});
}
// The largest pair of this block's partition that is strictly below `lim` (all threads; counts and keys of
// SWEEP_UNROLL slots per thread in flight, no dependent loads).  Result in *s_out; s_warp: 32 Best of scratch.
__device__ __forceinline__ void sweep_below(const LoopArgs &a, uint64_t pbase, uint32_t R, const Best lim, Best *s_warp, Best *s_out) {
  Best b{0, 0, 0};
  for (uint32_t i0 = threadIdx.x; i0 < R; i0 += blockDim.x * SWEEP_UNROLL) {
    unsigned long long c[SWEEP_UNROLL], k[SWEEP_UNROLL];
#pragma unroll
    for (int u = 0; u < SWEEP_UNROLL; u++) {
      const uint32_t i = i0 + (uint32_t)u * blockDim.x;
      c[u] = i < R ? __ldcg(a.tab.cnts + pbase + i) : 0ull;
      k[u] = i < R ? __ldcg(a.tab.keys + pbase + i) : 0ull;
    }
#pragma unroll
    for (int u = 0; u < SWEEP_UNROLL; u++) {
      if (c[u] == 0 || c[u] < b.c || c[u] > lim.c) continue;
      const Best cand{c[u], pair_prio((uint32_t)(k[u] >> 32), (uint32_t)k[u]), pbase + i0 + (uint64_t)u * blockDim.x};
      if (!better(lim, cand)) continue;
      if (better(cand, b)) b = cand;
    }
  }
  block_best(b, s_warp, s_out);
}

// A work item of the drain: place `e` of segment j = (sender rank sd, block b); e == ~0u: no item.  cnt_off / plc_off:
// byte offsets of its count word (in this block's row) and of its place inside the sender's {XqHdr, segments} slot.
struct DrainItem { uint32_t e, j, sd, cnt_off, plc_off; };
__device__ __forceinline__ DrainItem drain_item(const LoopArgs &a, uint32_t item, uint32_t nseg) {
  DrainItem d;
  d.e = ~0u; d.j = 0; d.sd = 0; d.cnt_off = 0; d.plc_off = 0;
  if (item >= nseg * a.drain_places) return d;
  d.e = item / nseg;
  d.j = item - d.e * nseg;
  d.sd = d.j / a.xq.nblocks;
  const uint32_t b = d.j - d.sd * a.xq.nblocks;
  d.cnt_off = d.sd == a.xq.me ? (uint32_t)(offsetof(XqHdr, counts) + ((size_t)blockIdx.x * XQ_MAX_BLOCKS + b) * 8)
                              : (uint32_t)(offsetof(XqHdr, shared) + (size_t)b * 8);
  d.plc_off = (uint32_t)(offsetof(XqHdr, places) + ((size_t)d.e * XQ_MAX_BLOCKS + b) * 16);
  return d;
}
// What a drained entry needs (merge_loop_kernel): the front, the round's new pairs, the parked list, the partition.
struct FrontCtx {
  unsigned long long *fk, *fc, *nk, *nc, *ownk;
  long long *ownd;
  unsigned long long *nsk;
  uint32_t *nlist, *s_nocc, *s_own_n, *s_refresh, *s_povf, *s_occ, *s_lost;
  uint32_t own_base, z, part, newp_limit;
  uint64_t pbase;
  PairTab tab;
};
// One drained entry.  (Tried out of line, to shrink the loop: the calls and the context struct in local memory made the
// drain slower.)
__device__ __forceinline__ void front_take(const FrontCtx &f, unsigned long long key, long long delta) {
  const uint64_t hh = mix64(key);
  const uint32_t fs = smem_tab_find(f.fk, FRONT_SLOTS - 1, hh, key);
  unsigned long long *cnt = nullptr;   // the count this entry changes: a member of the front, or a new pair of this round
  if (fs != ~0u) cnt = f.fc + fs;
  else if ((uint32_t)(key >> 32) == f.z || (uint32_t)key == f.z) {   // a pair of the new token: cannot be in the front yet
    // Every new pair is counted twice: exactly, in the table of the round (nk / nc) as long as it has room, and in a
    // hash-bucket sketch that always has.  A round with more new pairs than the table takes (a frequent token next to
    // thousands of different neighbours) discards the table — WHICH pairs found room depends on the order of arrival and
    // differs between blocks — and raises the bound of the front to the largest bucket instead: an upper bound of every
    // new pair's count, the same in every block.  Exact: the invariant is "every pair outside the front is below the bound".
    smem_add64(f.nsk + ((uint32_t)(hh >> 12) & (NEWP_SKETCH - 1)), (unsigned long long)delta);
    if (*reinterpret_cast<volatile uint32_t *>(f.s_lost) == 0) {   // (once the round is lost its table is dead weight)
      const uint32_t ns = smem_tab_slot(f.nk, NEWP_SLOTS - 1, hh, key, f.s_nocc, f.nlist, f.newp_limit);
      if (ns != ~0u) cnt = f.nc + ns;
      else *f.s_lost = 1;
    }
  }
  if (cnt) smem_add64(cnt, (unsigned long long)delta);
  if (pair_part(f.tab, hh) == f.part) {
    const uint32_t q = atomicAdd(f.s_own_n, 1u) - f.own_base;
    if (q < OWN_CAP) { f.ownk[q] = key; f.ownd[q] = delta; }
    else {   // the list is full: straight into the partition
      uint64_t slot = ~0ull;
      if (pair_add_at(f.tab, f.pbase, (uint32_t)hh & f.tab.rmask, key, delta, &slot)) atomicAdd(f.s_occ, 1u);
      if (slot == ~0ull) *f.s_povf = 1;
    }
  }
}
// parked entries -> the partition (all threads of the block)
__device__ __forceinline__ void front_flush(const FrontCtx &f, uint32_t n) {
  uint32_t added = 0;
  for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) {
    const unsigned long long key = f.ownk[i];
    uint64_t slot = ~0ull;
    added += pair_add_at(f.tab, f.pbase, (uint32_t)mix64(key) & f.tab.rmask, key, f.ownd[i], &slot) ? 1u : 0u;
    if (slot == ~0ull) *f.s_povf = 1;   // this partition ran full: an update was lost (benign race: every writer stores 1)
  }
  if (added) atomicAdd(f.s_occ, added);
}

// 512 threads at most: 128 registers per thread (with 1024 threads and 64 registers the loop spilled and ran slower)
__global__ void __launch_bounds__(512, 1) merge_loop_kernel(LoopArgs a) {
  __shared__ Best s_warp[32];
  __shared__ Best s_bound, s_tmp;   // the bound of the front / scratch of a refresh
  __shared__ uint32_t s_dead;   // token slots of this block tombstoned in this launch
  __shared__ uint32_t s_defer_n, s_direct, s_out_n, s_occ, s_xf, s_povf, s_focc, s_nocc, s_own_n, s_refresh, s_lost, s_scan[33];
  __shared__ unsigned long long s_lostmax;
  const bool sys = a.xq.world > 1;
  // dynamic shared memory: [segment prefix: XQ_MAX_WORLD * XQ_MAX_BLOCKS + 4 words][claim bitmaps][front keys, counts]
  // [new-pair keys, counts][parked keys, deltas][new-pair slot list][tile tokens][tile offsets][word frequencies]
  uint32_t *s_pref = yt_dyn_smem;
  uint32_t *s_claim = s_pref + (XQ_MAX_WORLD * XQ_MAX_BLOCKS + 4);  // 2 bitmaps of CLAIM_WORDS x 32 flags
  unsigned long long *fk = reinterpret_cast<unsigned long long *>(s_claim + 2 * CLAIM_WORDS);
  unsigned long long *fc = fk + FRONT_SLOTS;
  unsigned long long *nk = fc + FRONT_SLOTS;
  unsigned long long *nc = nk + NEWP_SLOTS;
  unsigned long long *ownk = nc + NEWP_SLOTS;
  long long *ownd = reinterpret_cast<long long *>(ownk + OWN_CAP);
  uint32_t *nlist = reinterpret_cast<uint32_t *>(ownd + OWN_CAP);   // slots of nk taken in this round
  uint32_t *flist = nlist + NEWP_SLOTS;                              // slots of fk taken since the last refresh
  unsigned long long *nsk = reinterpret_cast<unsigned long long *>(flist + FRONT_LIST);   // sketch of the round's new pairs
  uint32_t *stok = reinterpret_cast<uint32_t *>(nsk + NEWP_SKETCH);
  uint32_t *soff = stok + a.smem_tok_cap;
  // RESIDENT only: word frequencies behind the offsets (8-byte aligned: both caps are even)
  unsigned long long *sfreq = reinterpret_cast<unsigned long long *>(soff + a.smem_word_cap + 2);
  for (uint32_t i = threadIdx.x; i < 2 * CLAIM_WORDS; i += blockDim.x) s_claim[i] = 0;
  for (uint32_t i = threadIdx.x; i < NEWP_SLOTS; i += blockDim.x) { nk[i] = PK_EMPTY; nc[i] = 0; }
  for (uint32_t i = threadIdx.x; i < NEWP_SKETCH; i += blockDim.x) nsk[i] = 0;
  // STREAMING carve of the same region: NSTAGE stages of (tokens, offsets), each 16-byte aligned;
  // full[s]: TMA bytes landed (tx count), empty[s]: all consumer warps are done with stage s
  __shared__ __align__(8) unsigned long long s_full[MAX_STAGES], s_empty[MAX_STAGES];
  const uint32_t n_stage = a.n_stage;
  const uint32_t stage_words = a.stream_tok_cap + a.stream_word_cap;  // uint32 per stage
  if (!a.resident && threadIdx.x == 0) {
    for (uint32_t st = 0; st < n_stage; st++) { mbar_init(&s_full[st], 1); mbar_init(&s_empty[st], (blockDim.x >> 5) - 1);  /* consumer warps */ }
#ifndef YT_SIMT_EMU
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
#endif
  }
  // STREAMING pipeline state of this thread (producer lane: empty-phase bits, consumers: full-phase bits)
  uint32_t pipe_used = 0, pipe_phase = 0, pipe_stage = 0;
  const uint64_t gtid = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const unsigned lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nwarp = blockDim.x >> 5;
  const uint32_t R = a.tab.rmask + 1;
  const uint64_t pbase = (uint64_t)blockIdx.x * R;  // this block's partition of the pair table
  const uint32_t n_done0 = a.ctl->n_done;
  uint32_t round = a.ctl->xq_round;                   // exchange rounds completed so far (same on every rank)
  unsigned long long tacc0 = 0, tacc1 = 0, tacc2 = 0, tacc3 = 0, titers = 0;  // phase timers (block 0, thread 0)

  // occupancy of this block's partition (keys never leave the table between rebuilds)
  {
    uint32_t occ = 0;
    for (uint32_t i = threadIdx.x; i < R; i += blockDim.x) occ += __ldcg(a.tab.keys + pbase + i) != PK_EMPTY ? 1u : 0u;
    for (int o = 16; o > 0; o >>= 1) occ += __shfl_xor_sync(0xffffffffu, occ, o);
    if (threadIdx.x == 0) {
      s_occ = 0; s_xf = 0; s_dead = 0; s_focc = 0; s_nocc = 0; s_own_n = 0; s_refresh = 1; s_out_n = 0; s_lost = 0; s_lostmax = 0;
      s_povf = __ldcg(a.tab.overflow) ? 1u : 0u;
      s_bound = Best{0, 0, 0};
    }
    __syncthreads();
    if (lane == 0 && occ) atomicAdd(&s_occ, occ);
  }

  // resident mode: this block's tile moves into shared memory once
  uint32_t rw0 = 0, rw1 = 0;
  unsigned long long my_slots = 0;   // token slots this block owns (for its compaction wish)
  if (a.resident && blockIdx.x < a.n_tiles) {
    rw0 = a.tile_desc[blockIdx.x].x;
    rw1 = a.tile_desc[blockIdx.x + 1].x;
    my_slots = a.tile_desc[blockIdx.x + 1].y - a.tile_desc[blockIdx.x].y;
    if (rw1 > rw0) {
      load_tile(a, rw0, rw1, stok, soff);
      for (uint32_t i = threadIdx.x; i < rw1 - rw0; i += blockDim.x) sfreq[i] = a.freq[rw0 + i];
    }
  } else if (!a.resident && a.n_tiles) {
    const uint32_t per_block = (a.n_tiles + gridDim.x - 1) / gridDim.x;
    const uint32_t k0 = min(a.n_tiles, blockIdx.x * per_block), k1 = min(a.n_tiles, k0 + per_block);
    my_slots = a.tile_desc[k1].y - a.tile_desc[k0].y;
  }
  uint32_t n_refresh = 0, fseq = 0;  // refreshes of this launch (block-uniform)
  __syncthreads();

  // parked entries -> this block's partition (all threads; leaves the list empty).  The list counter s_own_n only grows:
  // entry q sits at place q - own_base (no reset, hence no barrier between a flush and the next round's parking).
  FrontCtx fx;
  fx.fk = fk; fx.fc = fc; fx.nk = nk; fx.nc = nc; fx.ownk = ownk; fx.ownd = ownd; fx.nlist = nlist;
  fx.s_nocc = &s_nocc; fx.s_own_n = &s_own_n; fx.s_refresh = &s_refresh; fx.s_povf = &s_povf; fx.s_occ = &s_occ;
  fx.nsk = nsk; fx.s_lost = &s_lost; fx.newp_limit = a.newp_limit;
  fx.own_base = 0; fx.z = 0; fx.part = blockIdx.x; fx.pbase = pbase; fx.tab = a.tab;
  DrainItem ditem[DRAIN_ITEMS];   // this thread's items of the first trip of the drain
#pragma unroll
  for (int k = 0; k < DRAIN_ITEMS; k++) ditem[k] = drain_item(a, threadIdx.x + (uint32_t)k * blockDim.x, a.xq.world * a.xq.nblocks);
  auto flush_own = [&]() {
    __syncthreads();
    const uint32_t end = s_own_n, n = min(end - fx.own_base, OWN_CAP);
    fx.own_base = end;
    front_flush(fx, n);
    __syncthreads();
  };
  // the largest member of the front (.slot = its slot in the front), in every thread; one block barrier
  auto select = [&]() {
    Best b{0, 0, 0};
    const uint32_t nm = s_focc;   // members (<= FRONT_LIST)
    for (uint32_t q = threadIdx.x; q < nm; q += blockDim.x) {
      const uint32_t i = flist[q];
      const unsigned long long c = fc[i];
      if (c == 0 || c < b.c) continue;
      const unsigned long long k = fk[i];
      const Best cand{c, pair_prio((uint32_t)(k >> 32), (uint32_t)k), i};
      if (better(cand, b)) b = cand;
    }
    return block_best_all(b, s_warp);
  };
  // rebuild the front from the partitions (see above); every block of this GPU runs it in the same iteration
  auto refresh = [&]() {
    flush_own();
    fseq++;
    n_refresh++;
    unsigned long long *gdata = a.frontbuf + (size_t)gridDim.x * 16;
    unsigned long long *mine = gdata + (size_t)blockIdx.x * FRONT_TOP * 2;
    for (uint32_t i = threadIdx.x; i < FRONT_SLOTS; i += blockDim.x) { fk[i] = PK_EMPTY; fc[i] = 0; }
    for (uint32_t i = threadIdx.x; i < NEWP_SKETCH; i += blockDim.x) nsk[i] = 0;   // (the new bound covers every pair of the table)
    Best lim{~0ull, ~0ull, 0};
    int k = 0;
    for (; k < (int)a.front_top; k++) {
      sweep_below(a, pbase, R, lim, s_warp, &s_tmp);
      const Best t = s_tmp;
      if (t.c == 0) break;   // block-uniform
      if (threadIdx.x == 0) { st_relaxed(mine + 2 * k, t.c); st_relaxed(mine + 2 * k + 1, prio_key(t.prio)); }
      lim = t;
    }
    if (threadIdx.x == 0) {
      for (int q = k; q < FRONT_TOP; q++) { st_relaxed(mine + 2 * q, 0ull); st_relaxed(mine + 2 * q + 1, 0ull); }
      s_focc = 0; s_refresh = 0;
      st_release(a.frontbuf + (size_t)blockIdx.x * 16, (unsigned long long)fseq, false);   // orders the stores above
    }
    {
      unsigned long long t0 = 0;
      for (unsigned j = threadIdx.x; j < gridDim.x; j += blockDim.x)
        for (uint32_t spin = 0; ld_acquire(a.frontbuf + (size_t)j * 16, false) != (unsigned long long)fseq; spin++)
          spin_step(spin, t0, a.spin_limit_ns);
    }
    __syncthreads();
    Best bd{0, 0, 0};   // the bound: the last pair of every list that is full (a shorter list holds its whole partition)
    for (unsigned j = threadIdx.x; j < gridDim.x; j += blockDim.x) {
      const unsigned long long c = ld_relaxed(gdata + ((size_t)j * FRONT_TOP + a.front_top - 1) * 2);
      const unsigned long long key = ld_relaxed(gdata + ((size_t)j * FRONT_TOP + a.front_top - 1) * 2 + 1);
      if (!c) continue;
      const Best cand{c, pair_prio((uint32_t)(key >> 32), (uint32_t)key), 0};
      if (better(cand, bd)) bd = cand;
    }
    for (unsigned e = threadIdx.x; e < gridDim.x * FRONT_TOP; e += blockDim.x) {
      const unsigned long long c = ld_relaxed(gdata + (size_t)e * 2), key = ld_relaxed(gdata + (size_t)e * 2 + 1);
      if (c) smem_tab_add(fk, fc, FRONT_SLOTS - 1, mix64(key), key, (long long)c, &s_focc, flist);   // nblocks x FRONT_TOP <= FRONT_FILL
    }
    block_best(bd, s_warp, &s_bound);
  };

  for (uint32_t it = 0; it <= a.max_iters; ++it) {
    const uint32_t n_done = n_done0 + it;
    unsigned long long tq0 = gtid == 0 ? gtimer() : 0, tq1 = 0, tq2 = 0, tq2b = 0, tq3 = 0;
    // ---------------- uniform exit checks: the flags every block read off the last round's count words
    const uint32_t xf = s_xf;
    {
      uint32_t stop = 0, why = 0;
      if (xf & XQF_PLIMIT) why |= 1u;                               // a partition reached the load limit: rebuild (dead keys vanish)
      if (xf & XQF_OVERFLOW) why |= 2u;                             // lost count changes: rebuild from the tokens
      if (xf & XQF_PFULL) why |= 4u;                                // a partition ran full: grow the table
      if (n_done >= a.max_total || it == a.max_iters) stop = 4;     // done (or launch budget spent)
      else if (why) stop = 2;
      else if (xf & XQF_COMPACT) stop = 3;                          // some block wants a compaction
      if (stop) {
        if (gtid == 0) { a.ctl->stop = stop == 4 ? 0u : stop; a.ctl->stop_why = why; }
        break;
      }
    }
    // ---------------- elect the pair from the front (no communication)
    Best win;
    for (bool need = s_refresh || s_focc > FRONT_FILL;; need = true) {   // at most two trips: "the front is exhausted" shows in the election
      if (need) refresh();
      win = select();
      if (need || !(win.c == 0 || better(s_bound, win))) break;
      __syncthreads();   // (s_warp of the election is free again)
    }
    if (win.c == 0) {                                               // no pair left (bpe.cpp:1137-1145)
      if (gtid == 0) { a.ctl->stop = 1; a.ctl->stop_why = 0; }
      break;
    }
    MergeOp op;
    op.key = fk[win.slot];
    op.x = (uint32_t)(op.key >> 32);
    op.y = (uint32_t)op.key;
    op.z = a.first_new_id + n_done;
    if (gtid == 0) {
      a.rules[3 * n_done + 0] = op.x; a.rules[3 * n_done + 1] = op.y; a.rules[3 * n_done + 2] = op.z;
      a.rfreq[n_done] = win.c;
      a.ctl->n_done = n_done + 1;
    }
    if (gtid == 0) tq1 = gtimer();
    // every occurrence of (x,y) is merged below and no count changes are emitted for it: the front drops it here, its
    // owner parks the matching update of the partition (the front's count is exact)
    if (threadIdx.x == 0) {   // (no barrier needed behind this: the apply phase touches none of it)
      fc[win.slot] = 0;
      s_nocc = 0;             // last read in the previous iteration's fold, next written in this iteration's drain
      if (pair_part(a.tab, mix64(op.key)) == blockIdx.x) {
        const uint32_t q = s_own_n++ - fx.own_base;   // (only thread 0 touches the list between the drain and flush_own)
        if (q < OWN_CAP) { ownk[q] = op.key; ownd[q] = -(long long)win.c; }
        else pair_add_at(a.tab, pbase, (uint32_t)mix64(op.key) & a.tab.rmask, op.key, -(long long)win.c);
      }
    }
    // ---------------- apply x y -> z: count changes go to this block's segment of round + 1 (on every rank)
    const uint32_t nround = round + 1;
    XqOut xo;
    xo.off = xq_seg_off(a.xq, nround & 1u, a.xq.me, blockIdx.x);
    xo.s_n = &s_out_n;
    xo.stamp = nround % XQ_STAMP_MOD;
    xo.parity = nround & 1u;
    unsigned long long dead = 0;
    if (a.resident) {
      if (rw1 > rw0) dead = process_tile(stok, soff, rw1 - rw0, soff[rw1 - rw0], s_claim,
                                           reinterpret_cast<const uint64_t *>(sfreq), op, a, xo);
    } else {
      // STREAMING: this block owns a contiguous chunk of tiles that flows through an n_stage ring of
      // shared-memory stages.  Lane 0 of warp 0 is the PRODUCER: it keeps up to n_stage tiles in
      // flight with TMA bulk copies (tokens + offsets, 16-byte aligned windows, completion on
      // full[s]) and refills a stage as soon as all consumer warps have released it (empty[s]).
      // Warps 1.. are CONSUMERS: they scan a tile out of shared memory token-parallel and append
      // the words that hold (x,y) to the block's deferred list; no block barrier in the tile loop.
      // The deferred words are rewritten afterwards straight in HBM, one warp per word, so their
      // latencies overlap each other instead of stalling the copy pipeline.
      const uint32_t per_block = (a.n_tiles + gridDim.x - 1) / gridDim.x;
      const uint32_t k_first = min(a.n_tiles, blockIdx.x * per_block);
      const uint32_t my_tiles = min(a.n_tiles, k_first + per_block) - k_first;
      uint4 *defer = a.defer + (size_t)blockIdx.x * a.defer_cap;
      if (threadIdx.x == 0) { s_defer_n = 0; s_direct = 0; }
      __syncthreads();
      auto staged = [&](uint2 d0, uint2 d1) {  // does this tile go through shared memory?
        return d1.x > d0.x && win_bytes(d0.y, d1.y) <= a.stream_tok_cap * 4u &&
               win_bytes(d0.x, d1.x + 1) <= a.stream_word_cap * 4u;
      };
      // tile descriptors travel in lane-distributed batches: lane j of a warp holds tile_desc[base + j],
      // tiles base .. base+30 take (d0, d1) from lanes (j, j+1) by shuffle, so the L2 latency of the
      // descriptor loads is paid once per 31 tiles instead of once per tile
      auto load_batch = [&](uint32_t base) {
        const uint32_t idx = min(k_first + base + lane, k_first + my_tiles);
        return a.tile_desc[idx];
      };
      if (wid == 0) {
        uint32_t used = pipe_used, ephase = pipe_phase, st = pipe_stage;  // barrier phases persist across merges
        uint2 batch = make_uint2(0, 0);
        for (uint32_t t = 0; t < my_tiles; t++) {
          const uint32_t j = t % 31;
          if (j == 0) batch = load_batch(t);
          uint2 d0, d1;
          tile_pair(batch, j, d0, d1);
          if (!staged(d0, d1)) continue;
          if (lane == 0) {
            if ((used >> st) & 1u) mbar_wait(&s_empty[st], (ephase >> st) & 1u);
            uint32_t *dst = stok + st * stage_words;
            const uint32_t bt = win_bytes(d0.y, d1.y), bo = win_bytes(d0.x, d1.x + 1);
            mbar_expect_tx(&s_full[st], bt + bo);
            tma_bulk_g2s(dst, a.tok + win_lo(d0.y), bt, &s_full[st]);
            tma_bulk_g2s(dst + a.stream_tok_cap, a.off + win_lo(d0.x), bo, &s_full[st]);
          }
          if ((used >> st) & 1u) ephase ^= 1u << st;
          used |= 1u << st;
          st = st + 1 == n_stage ? 0 : st + 1;
          __syncwarp();
        }
        pipe_used = used; pipe_phase = ephase; pipe_stage = st;
      } else {
        uint32_t fphase = pipe_phase, st = pipe_stage;
        const unsigned cw = wid - 1, ncw = nwarp - 1;  // consumer warp index / count
        uint2 batch = make_uint2(0, 0);
        for (uint32_t t = 0; t < my_tiles; t++) {
          const uint32_t j = t % 31;
          if (j == 0) batch = load_batch(t);
          uint2 d0, d1;
          tile_pair(batch, j, d0, d1);
          if (d1.x <= d0.x) continue;
          if (!staged(d0, d1)) { if (cw == 0 && lane == 0) s_direct = 1; continue; }  // oversized: direct pass below
          mbar_wait(&s_full[st], (fphase >> st) & 1u);
          fphase ^= 1u << st;
          const uint32_t *stg = stok + st * stage_words;     // 16-byte aligned window of the stage
          const uint32_t head = d0.y - win_lo(d0.y);         // 0..3 tokens of the previous tile in front
          const uint32_t *tk = stg + head;
          const uint32_t *of = stg + a.stream_tok_cap + (d0.x - win_lo(d0.x));
          const uint32_t span = d1.y - d0.y, nw = d1.x - d0.x, obase = d0.y;
          auto report = [&](uint32_t i) {  // token i of the tile starts an (x,y) occurrence
            const uint32_t lo = word_at(of, nw, i, obase);
            const uint32_t o = of[lo] - obase, wcap = of[lo + 1] - obase - o;
            for (uint32_t q2 = o; q2 < i; q2++)  // only the first hit of a word reports it
              if (tk[q2] == op.x && tk[q2 + 1] == op.y) return;
            const uint32_t slot = atomicAdd(&s_defer_n, 1u);
            if (slot < a.defer_cap) defer[slot] = make_uint4(d0.x + lo, obase + o, wcap, 0u);
            else s_direct = 1;  // list full: the direct pass below picks the rest up
          };
          // eight tokens per lane from two 16-byte shared loads; the token after them comes from the
          // next lane.  p = position in the aligned window; occurrence p is inside the tile iff
          // head <= p and p + 1 < total (a word-initial token is never y, so none straddles tiles).
          // 8 tokens per lane: a scalar scan left most of the HBM bandwidth unused.
          const uint32_t total = head + span;
          for (uint32_t base = cw * 256; base < total; base += ncw * 256) {
            const uint32_t p = base + lane * 8;
            uint4 v = make_uint4(~0u, ~0u, ~0u, ~0u), u = v;
            if (p < total) v = *reinterpret_cast<const uint4 *>(stg + p);
            if (p + 4 < total) u = *reinterpret_cast<const uint4 *>(stg + p + 4);
            uint32_t nxt = __shfl_down_sync(0xffffffffu, v.x, 1);
            if (lane == 31) nxt = p + 8 < total ? stg[p + 8] : ~0u;
            uint32_t m = match8(v, u, nxt, op);
            if (!__ballot_sync(0xffffffffu, m)) continue;
            while (m) {
              const uint32_t pk = p + (uint32_t)__ffs(m) - 1u;
              m &= m - 1u;
              if (pk >= head && pk + 1 < total) report(pk - head);
            }
          }
          __syncwarp();
          if (lane == 0) mbar_arrive(&s_empty[st]);
          st = st + 1 == n_stage ? 0 : st + 1;
        }
        pipe_phase = fphase; pipe_stage = st;
      }
      __syncthreads();
      {
        const uint32_t n_def = min(s_defer_n, a.defer_cap);
        for (uint32_t j = wid; j < n_def; j += nwarp) {
          const uint4 e = defer[j];
          const long long f = (long long)a.freq[e.x];
          const uint32_t merges = warp_apply_word(a.tok + e.y, e.z, nullptr, f, op, lane, a, xo);
          if (lane == 0) dead += merges;
        }
        if (s_direct && my_tiles) {  // oversized tiles / overflowed list: exact thread-per-word pass on global memory
          __syncthreads();
          const uint32_t w_lo = a.tile_desc[k_first].x, w_hi = a.tile_desc[k_first + my_tiles].x;
          dead += process_tile_direct(a.tok, a.off, a.freq, w_lo, w_hi, op, a, xo);
        }
      }
      // write-through stores (generic proxy) must be ordered before the next iteration's bulk loads
#ifndef YT_SIMT_EMU
      asm volatile("fence.proxy.async;" ::: "memory");
#endif
    
    }
    for (int o = 16; o > 0; o >>= 1) dead += __shfl_xor_sync(0xffffffffu, dead, o);
    if (lane == 0 && dead) atomicAdd(&s_dead, (uint32_t)dead);
    __syncthreads();  // all entries of this block are on their way
    {
      // the count word of this segment, into the row of every local block and once into every other rank (every thread
      // computes the same word and stores a share).  No fence: the entries carry their own stamps, the count word may overtake them.
      const uint32_t n = s_out_n;
      uint32_t word = n > a.xq.seg_cap ? (a.xq.seg_cap | XQ_CNT_OVF) : n;
      if ((unsigned long long)s_dead * 4 > my_slots && my_slots > a.dead_min_slots) word |= XQ_CNT_COMPACT;   // s_dead: tombstoned in this launch
      if (s_occ > a.part_limit) word |= XQ_CNT_PLIMIT;   // state of the partition as of the last flush
      if (s_povf) word |= XQ_CNT_PFULL;
      const unsigned long long cw = ((unsigned long long)nround << 32) | word;
      // local readers: one word per reader block (its private row); the other ranks: one word per rank
      for (uint32_t rb = threadIdx.x; rb < a.xq.nblocks; rb += blockDim.x)
        st_relaxed_any(xq_cnt(xq_hdr(a.xq, a.xq.me, nround & 1u, a.xq.me), rb, blockIdx.x), cw, false);
      if (threadIdx.x < a.xq.world && threadIdx.x != a.xq.me)
        st_relaxed_any(&xq_hdr(a.xq, threadIdx.x, nround & 1u, a.xq.me)->shared[blockIdx.x], cw, true);
      if (threadIdx.x == 0) s_xf = 0;   // accumulator of the poll below
    }
    if (gtid == 0) tq2 = gtimer();
    round = nround;
    // ---------------- while the other blocks finish their apply phase: the parked entries of the previous round (and
    // the consumed pair) go into this block's partition
    flush_own();
    if (threadIdx.x == 0) s_out_n = 0;   // (read by all before flush_own's barriers; next used in the next apply phase)
    if (gtid == 0) tq2b = gtimer();
    // ---------------- drain: the count changes of this merge, from every block of every GPU.  Thread j polls the count
    // word of segment j (barrier and count fetch in one) and, when the segment is short, fetches and handles its entries
    // right away — no block barrier sits between the arrival of a count word and the loads of its entries; longer
    // segments (the first rounds of a run) are shared by the whole block afterwards.
    {
      fx.z = op.z;
      const uint32_t nseg = a.xq.world * a.xq.nblocks, parity = round & 1u, stamp = round % XQ_STAMP_MOD;
      uint32_t flags = 0, big = 0;
      unsigned long long t0 = 0;
      // One work item per (place e, segment j), numbered place-major: item = e * nseg + j.  The thread of an item polls
      // the count word of segment j in this block's row and loads place e of that segment from the matrix — consecutive
      // lanes touch consecutive words / slots, and the entries of a round spread over the whole block.  No barrier between
      // the arrival of a count word and the handling of its entries.  DRAIN_ITEMS items per thread and trip, their loads
      // all in flight.  (Versions measured before this one: thread j handling all places of sender j — the entry
      // handlers of a warp's 32 senders ran one after the other; one private 128-byte line per (reader, sender) — every
      // lane on its own line, 64 cycles of load/store unit per warp instruction, polled: 1 us per sweep.)
      {
        const uint32_t nitems = nseg * a.drain_places;
        const unsigned char *region = xq_base(a.xq, a.xq.me) + (size_t)parity * a.xq.world * a.xq.per_sender;   // [sender]{XqHdr, segments} of this parity
        for (uint32_t base = threadIdx.x, trip = 0; base < nitems; base += (uint32_t)DRAIN_ITEMS * blockDim.x, trip++) {   // (one trip: 1 GPU, >= 352 threads)
          uint32_t ie[DRAIN_ITEMS], ij[DRAIN_ITEMS];
          const unsigned long long *wp[DRAIN_ITEMS], *ep[DRAIN_ITEMS];
          unsigned long long hv[DRAIN_ITEMS], e0 = 0, e1 = 0;
#pragma unroll
          for (int k = 0; k < DRAIN_ITEMS; k++) {
            DrainItem di = ditem[k];   // first trip: decoded once per launch (the divisions cost ~25 instructions each)
            if (trip) di = drain_item(a, base + (uint32_t)k * blockDim.x, nseg);
            ie[k] = di.e; ij[k] = di.j;
            const unsigned char *h = region + (size_t)di.sd * a.xq.per_sender;
            wp[k] = reinterpret_cast<const unsigned long long *>(h + di.cnt_off);
            ep[k] = reinterpret_cast<const unsigned long long *>(h + di.plc_off);
            hv[k] = di.e != ~0u ? ld_relaxed_any(wp[k], sys) : 0ull;
          }
          if (ie[0] != ~0u) ld_relaxed2(ep[0], &e0, &e1, sys);   // speculative: places 0 .. 2 (3) usually hold an entry
#pragma unroll
          for (int k = 0; k < DRAIN_ITEMS; k++) {
            if (ie[k] == ~0u) continue;
            const uint32_t e = ie[k], j = ij[k];
            for (uint32_t spin = 0; (uint32_t)(hv[k] >> 32) != round; spin++) {
              spin_step(spin, t0, a.spin_limit_ns);
              hv[k] = ld_relaxed_any(wp[k], sys);
              if (k == 0) ld_relaxed2(ep[0], &e0, &e1, sys);
            }
            const uint32_t c = (uint32_t)hv[k];
            uint32_t n = c & XQ_CNT_MASK;
            if (n > a.xq.seg_cap) n = a.xq.seg_cap;
            if (e == 0) {   // the place-0 thread speaks for the segment
              cnt_flags(flags, c, false);
              const uint32_t nb = n < a.drain_places ? n : a.drain_places;
              s_pref[j] = n - nb;   // the rest: the shared walk below (place matrix up to XQ_BOX, then the sender's segment)
              if (n > nb) big = 1;
            }
            if (e >= n) continue;
            if (k != 0) ld_relaxed2(ep[k], &e0, &e1, sys);   // the later items of a thread are the rarely used places
            unsigned long long key = 0;
            long long delta = 0;
            for (uint32_t spin = 0; !xq_unpack(e0, e1, stamp, &key, &delta); spin++) {   // the count word overtook the entry
              spin_step(spin, t0, a.spin_limit_ns);
              ld_relaxed2(ep[k], &e0, &e1, sys);
            }
            front_take(fx, key, delta);
          }
        }
      }
      if (flags) atomicOr(&s_xf, flags);
      if (__syncthreads_or((int)big)) {   // block-uniform
        xq_prefix(a, s_pref, s_scan);
        const uint32_t total = s_pref[nseg];
        for (uint32_t i = threadIdx.x; i < total; i += blockDim.x) {
          unsigned long long key = 0;
          long long delta = 0;
          xq_entry(a, round, s_pref, i, &key, &delta, a.drain_places);
          front_take(fx, key, delta);
        }
      }
    }
    __syncthreads();
    // ---- the new token's pairs: those not below the bound join the front — or, in a round with more of them than
    // the table takes, all of them stay outside and the bound rises to the largest sketch bucket (front_take)
    if (s_nocc) {   // block-uniform (read after the barrier); 0: the round had no new pair
      const Best bd = s_bound;
      const uint32_t nn = min(s_nocc, NEWP_SLOTS);   // one list entry per slot taken
      const bool lost = s_lost != 0 || s_nocc > a.newp_limit;   // the same verdict in every block (distinct new pairs > limit)
      for (uint32_t q = threadIdx.x; q < nn; q += blockDim.x) {
        const uint32_t i = nlist[q];
        const unsigned long long k = nk[i];
        const unsigned long long c = nc[i];
        nk[i] = PK_EMPTY; nc[i] = 0;
        if (lost || (long long)c <= 0) continue;
        const Best cand{c, pair_prio((uint32_t)(k >> 32), (uint32_t)k), 0};
        if (better(bd, cand)) continue;
        if (!smem_tab_add(fk, fc, FRONT_SLOTS - 1, mix64(k), k, (long long)c, &s_focc, flist)) s_refresh = 1;
      }
      // The sketch is read and cleared only here, in a lost round (and cleared by every refresh): between two such
      // points its buckets keep adding up the new pairs of ALL rounds — still an upper bound of each of them (counts of
      // pairs outside the front only fall), a little looser, and the usual round pays nothing for it.
      if (lost) {
        unsigned long long m = 0;
        for (uint32_t i = threadIdx.x; i < NEWP_SKETCH; i += blockDim.x) { m = max(m, nsk[i]); nsk[i] = 0; }
        if (m) atomicMax(&s_lostmax, m);
        __syncthreads();
        if (threadIdx.x == 0) {
          const Best lb{s_lostmax, ~0ull, 0};
          if (better(lb, s_bound)) s_bound = lb;
          s_lost = 0; s_lostmax = 0;
        }
      }
    }
    __syncthreads();
    if (gtid == 0) {
      tq3 = gtimer();
      tacc1 += tq1 - tq0;   // election from the front (+ refreshes)
      tacc2 += tq2 - tq1;   // apply
      tacc3 += tq2b - tq2;  // parked entries -> partition
      tacc0 += tq3 - tq2b;  // drain + new pairs
      titers += 1;
    }
  }
  flush_own();   // every exit path: the partition is complete again
  if (threadIdx.x == 0 && s_povf) atomicExch(a.tab.overflow, 1u);
  if (gtid == 0 && n_refresh) atomicAdd(&a.ctl->n_sweeps, (unsigned long long)n_refresh);
  if (gtid == 0) {
    a.ctl->xq_round = round;
    a.ctl->t_phase[0] += tacc0; a.ctl->t_phase[1] += tacc1; a.ctl->t_phase[2] += tacc2; a.ctl->t_phase[3] += tacc3;
    a.ctl->iters += titers;
  }
  // resident tiles go back to HBM on every exit path
  __syncthreads();
  if (a.resident && rw1 > rw0) {
    const uint32_t o0 = a.off[rw0], span = a.off[rw1] - o0;
    for (uint32_t i = threadIdx.x; i < span; i += blockDim.x) a.tok[o0 + i] = stok[i];
  }
}

// ---- exchange rounds outside the loop (multi-GPU table build): one block per partition -----------
// xq_publish_table_kernel: block b enumerates the live (key, count) pairs of partition b of a SNAPSHOT of the local
// table in slot order and copies those numbered [chunk * seg_cap, (chunk + 1) * seg_cap) into segment b of round
// `round` on every OTHER rank, then stores its stamped count word everywhere (XQ_CNT_MORE: further chunks follow;
// XQ_CNT_OVF: the local histogram had overflowed - every rank retries with a larger table).
__global__ void __launch_bounds__(256) xq_publish_table_kernel(LoopArgs a, uint32_t round, uint32_t chunk, const uint32_t *local_overflow) {
  const uint32_t R = a.tab.rmask + 1;
  const uint64_t pbase = (uint64_t)blockIdx.x * R;
  const size_t off = xq_seg_off(a.xq, round & 1u, a.xq.me, blockIdx.x);
  const unsigned lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nwarp = blockDim.x >> 5;
  const uint64_t lo = (uint64_t)chunk * a.xq.seg_cap, hi = lo + a.xq.seg_cap;
  __shared__ uint32_t s_w[32];
  uint32_t done = 0;  // live pairs before this pass (block-uniform)
  for (uint32_t i0 = 0; i0 < R; i0 += blockDim.x) {  // block-uniform trip count, slot order
    const uint32_t i = i0 + threadIdx.x;
    unsigned long long k = PK_EMPTY, c = 0;
    if (i < R) { k = a.tab.keys[pbase + i]; c = a.tab.cnts[pbase + i]; }
    const bool has = k != PK_EMPTY && c != 0;
    const unsigned m = __ballot_sync(0xffffffffu, has);
    if (lane == 0) s_w[wid] = (uint32_t)__popc(m);
    __syncthreads();
    uint32_t before = 0, all = 0;
    for (unsigned w = 0; w < nwarp; w++) { const uint32_t v = s_w[w]; if (w < wid) before += v; all += v; }
    if (has) {
      const uint64_t idx = (uint64_t)done + before + __popc(m & ((1u << lane) - 1u));
      if (idx >= lo && idx < hi) {
        const uint4 e = xq_pack(round % XQ_STAMP_MOD, k, (long long)c);
#pragma unroll
        for (int d = 0; d < XQ_MAX_WORLD; d++)
          if ((uint32_t)d < a.xq.world && (uint32_t)d != a.xq.me) reinterpret_cast<uint4 *>(a.xq.base[d] + off)[idx - lo] = e;
      }
    }
    done += all;
    __syncthreads();
  }
  {
    const uint64_t total = done;
    uint32_t word = total > lo ? (uint32_t)(total - lo < (uint64_t)a.xq.seg_cap ? total - lo : (uint64_t)a.xq.seg_cap) : 0u;
    if (total > hi) word |= XQ_CNT_MORE;
    if (__ldcg(local_overflow)) word |= XQ_CNT_OVF;
    const unsigned long long cw = ((unsigned long long)round << 32) | word;
    const uint32_t nbox = a.xq.world * a.xq.nblocks;
    for (uint32_t t = threadIdx.x; t < nbox; t += blockDim.x) {
      const uint32_t d = t / a.xq.nblocks, rb = t - d * a.xq.nblocks;
      st_relaxed_any(xq_cnt(xq_hdr(a.xq, d, round & 1u, a.xq.me), rb, blockIdx.x), cw, true);
    }
  }
}
// xq_absorb_kernel: block b waits for round `round` of every block of every rank and adds the peers' pairs it owns
// to partition b of the live table.
__global__ void __launch_bounds__(256) xq_absorb_kernel(LoopArgs a, uint32_t round) {
  __shared__ uint32_t s_scan[33], s_occ, s_acc;
  uint32_t *s_pref = yt_dyn_smem;
  if (threadIdx.x == 0) { s_occ = 0; s_acc = 0; }
  __syncthreads();
  xq_poll_counts(a, round, true, s_pref, &s_acc);
  xq_drain(a, round, s_pref, s_scan, &s_occ);
  __syncthreads();
  if (threadIdx.x == 0) {
    if (s_acc) atomicOr(&a.ctl->xq_flags, s_acc);
    if (blockIdx.x == 0) a.ctl->xq_round = round;
  }
}

// ---- tile planning -----------------------------------------------------------------------------
// tile k = words whose first token slot lies in [k*q, (k+1)*q); tile_desc[k] = (its first word,
// that word's token offset); tile_desc[n_tiles] = (n_words, n_slots).
__global__ void tile_desc_kernel(const uint32_t *__restrict__ off, uint64_t n_words, uint32_t q, uint32_t n_tiles,
                                 uint2 *__restrict__ desc) {
  uint64_t w = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (w >= n_words) return;
  const uint32_t ow = off[w];
  const uint32_t k1 = ow / q;
  const int64_t k0 = w == 0 ? -1 : (int64_t)(off[w - 1] / q);
  for (int64_t k = k0 + 1; k <= (int64_t)k1; k++) desc[k] = make_uint2((uint32_t)w, ow);
  if (w + 1 == n_words)
    for (uint32_t k = k1 + 1; k <= n_tiles; k++) desc[k] = make_uint2((uint32_t)n_words, off[n_words]);
}
__global__ void tile_stats_kernel(const uint2 *__restrict__ desc, uint32_t n_tiles,
                                  uint32_t *out /* [0] max span, [1] max words */) {
  uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n_tiles) return;
  uint2 d0 = desc[k], d1 = desc[k + 1];
  if (d1.x <= d0.x) return;
  atomicMax(out, d1.y - d0.y);
  atomicMax(out + 1, d1.x - d0.x);
}
