// common.cuh — context, error plumbing, device buffers, stage timers shared by the CUDA units.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>
#include <climits>
#include <cstdlib>
#include <map>
#include <string>
#include <vector>

#include "../../include/yttm_b200.h"
#include "bpe_core.cuh"

namespace ytc {

struct DevBuf {  // a growable raw device allocation
  void *p = nullptr;
  size_t cap = 0;
  cudaError_t reserve(size_t bytes) {
    if (bytes <= cap) return cudaSuccess;
    if (p) cudaFree(p);
    p = nullptr; cap = 0;
    size_t want = bytes + bytes / 8 + 256;
    cudaError_t e = cudaMalloc(&p, want);
    if (e == cudaSuccess) cap = want;
    return e;
  }
  void release() { if (p) cudaFree(p); p = nullptr; cap = 0; }
  template <class T> T *as() const { return reinterpret_cast<T *>(p); }
};

struct StageTimer { cudaEvent_t a = nullptr, b = nullptr; float ms = -1.f; bool pending = false; };

}  // namespace ytc

// Merge-loop control block in device memory (read back by the host after each launch).
struct YtLoopCtl {
  uint32_t n_done;            // merges recorded so far
  uint32_t stop;              // 0 running, 1 no pair left, 2 table wants rebuild, 3 compaction wanted
  uint32_t n_keys;            // occupied slots of the pair table
  uint32_t overflow;          // a probe sequence wrapped (fatal)
  unsigned long long dead;    // token slots tombstoned since the last compaction
  unsigned long long slots;   // token slots at the last compaction
  unsigned long long t_phase[4];  // ns spent by block 0 in: [0] drain (wait for the count words, entries, new pairs),
                                  // [1] election (+ refreshes), [2] apply, [3] parked entries into its partition
  unsigned long long iters;       // iterations those times cover
  uint32_t xq_round;              // exchange rounds completed (same on every rank of the job)
  uint32_t stop_why;              // stop == 2: 1 partition nearly full, 2 exchange segment overflowed, 4 partition full, 8 load factor
  uint32_t xq_flags;              // flags of the peers' last out-of-loop round (xq_absorb_kernel)
  uint32_t max_part_occ;          // part_occ_kernel: fullest partition of the table
  unsigned long long n_sweeps;    // refreshes of the replicated front (merge_loop.cuh)
};

struct yttm_ctx {
  int device = 0;
  int n_sm = 0;
  cudaStream_t stream = nullptr;
  std::string err;
  uint64_t launches = 0;
  std::map<std::string, ytc::StageTimer> timers;

  // ---- corpus
  ytc::DevBuf text_buf;            // 16 pad bytes (spaces) + text + 32 pad bytes
  const uint8_t *d_text = nullptr; // first text byte
  uint64_t n_text = 0;
  bool text_external = false;

  // ---- char histogram / alphabet
  ytc::DevBuf hist;   // uint64[CP_LIMIT + 1]; last = data_len
  ytc::DevBuf cp2id;  // uint32[CP_LIMIT]
  std::vector<uint32_t> h_hist_cp;
  std::vector<uint64_t> h_hist_cnt;
  uint64_t data_len = 0;
  uint32_t space_id = 0;
  bool have_alphabet = false;
  // pipelined ingest (yttm_train_load_corpus): the histogram / the word table of the text were built while it was copied
  bool pipe_hist = false;
  uint64_t pipe_wtab_cap = 0;
  cudaStream_t stream2 = nullptr;
  cudaEvent_t ev_pipe = nullptr;

  // ---- word table / unique words
  ytc::DevBuf wkey, wcnt, wpos, wfreq, wlen, scan_tmp, counters;
  uint64_t n_word_occ = 0, n_unique = 0;

  // ---- fed corpus (yttm_train_feed_*): pieces cut on the host from two pinned staging buffers, copied on stream2 into
  // two device piece buffers; each piece's words (per-piece table wkey / wcnt) are merged into the persistent table
  // fkey / fcnt, whose words' bytes live in the arena (16 pad spaces + words, each followed by one space)
  bool feeding = false;         // between feed_begin and feed_end
  bool fed_words = false;       // the text is the arena of a fed corpus; wpos / wfreq / n_unique hold its words
  uint8_t *feed_stage[2] = {nullptr, nullptr};
  uint64_t feed_stage_cap[2] = {0, 0};
  int feed_cur = 0;             // staging buffer being filled
  uint64_t feed_len = 0;        // its bytes
  uint64_t feed_nows = 0;       // its first bytes known to hold no whitespace byte
  int feed_pending = -1;        // a piece copied but not yet processed (its staging / piece buffer index)
  uint64_t feed_pending_len = 0;
  uint64_t feed_piece = 0;      // nominal piece size
  ytc::DevBuf feed_dev[2], fkey, fcnt, arena;
  cudaEvent_t ev_feed_copied[2] = {nullptr, nullptr}, ev_feed_done[2] = {nullptr, nullptr};
  uint64_t feed_wcap = 0, feed_fcap = 0, feed_fn = 0;   // per-piece / persistent table slots, persistent words
  uint64_t arena_len = 0, n_fed = 0, feed_pieces = 0;
  uint64_t dev_peak = 0;        // largest sum of the DevBuf capacities of the current training

  // ---- packed words (double buffered for compaction)
  ytc::DevBuf tok[2], off[2], freq[2];
  int cur = 0;
  uint64_t n_words = 0;  // entries of off minus one
  uint64_t n_slots = 0;  // token slots

  // ---- pair table: p_nparts partitions of p_rmask + 1 slots (pcap = their product)
  ytc::DevBuf pkey, pcnt, scratch_key, scratch_cnt;
  uint64_t pcap = 0;
  uint32_t p_rmask = 0, p_nparts = 0;

  // ---- exchange buffer of the merge loop (merge_loop.cuh); world > 1: peers[] are the other ranks' regions
  ytc::DevBuf xq_buf, xq_arrive;
  uint32_t xq_world = 1, xq_me = 0, xq_seg_cap = 0, xq_nblocks = 0;
  uint64_t xq_per_sender = 0, xq_bytes = 0;
  void *xq_peer[8] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
  bool xq_peer_ipc[8] = {false, false, false, false, false, false, false, false};
  bool xq_connected = false;

  // ---- merge loop
  ytc::DevBuf ctl, frontbuf, d_rules, d_rfreq, tiles, defer;
  int loop_smem = 0, loop_resident = 0, loop_stages = 2;
  uint32_t loop_tok_cap = 0, loop_word_cap = 0, loop_stream_q = 0, loop_stream_tok_cap = 0, loop_stream_word_cap = 0;
  int loop_blocks = 0, loop_threads = 0;
  double loop_phase_ms[4] = {0, 0, 0, 0};   // YtLoopCtl::t_phase of the last yttm_train_run
  uint64_t loop_iters = 0, loop_relaunches = 0, loop_sweeps = 0;
  uint32_t loop_xq_round = 0;   // YtLoopCtl::xq_round after the last yttm_train_run
  double enc_chunks = -1;       // chunks the last host-buffer encode call was cut into (encode.cu)

  yttm_train_stats stats{};
};

extern thread_local std::string g_yttm_create_error;

// The environment knobs that fix a context's launch geometry and its exchange buffer when it first trains (train.cu;
// NULL-terminated): a cache of contexts must key on their values.  YT_EMU_SMS is the SM count of the CPU emulation used
// by the tests.
extern const char *const yttm_geometry_knobs[];

// exclusive scan of uint64 on the context stream (train.cu); *d_total receives the sum
int yttm_device_scan_u64(yttm_ctx *c, const unsigned long long *in, uint64_t n, unsigned long long *out,
                         unsigned long long *d_total);

// whether the host trainings (bpe_host.cpp) feed a corpus of n bytes (UINT64_MAX: unknown) instead of loading it (train.cu)
bool yttm_train_feed_selected(yttm_ctx *c, uint64_t n);

#define YT_CUDA(ctx, call)                                                                       \
  do {                                                                                           \
    cudaError_t e__ = (call);                                                                    \
    if (e__ != cudaSuccess) {                                                                    \
      (ctx)->err = std::string(#call) + ": " + cudaGetErrorString(e__) + " (" + __FILE__ + ":" + \
                   std::to_string(__LINE__) + ")";                                               \
      return 1;                                                                                  \
    }                                                                                            \
  } while (0)

#define YT_FAIL(ctx, msg)     \
  do {                        \
    (ctx)->err = (msg);       \
    return 1;                 \
  } while (0)

namespace ytc {
inline void timer_begin(yttm_ctx *c, const char *name) {
  StageTimer &t = c->timers[name];
  if (!t.a) { cudaEventCreate(&t.a); cudaEventCreate(&t.b); }
  cudaEventRecord(t.a, c->stream);
}
inline void timer_end(yttm_ctx *c, const char *name) {  // records only; timer_ms() resolves it
  StageTimer &t = c->timers[name];
  cudaEventRecord(t.b, c->stream);
  t.pending = true;
}
inline double timer_ms(yttm_ctx *c, const char *name) {
  auto it = c->timers.find(name);
  if (it == c->timers.end()) return -1.0;
  StageTimer &t = it->second;
  if (t.pending) {
    cudaEventSynchronize(t.b);
    cudaEventElapsedTime(&t.ms, t.a, t.b);
    t.pending = false;
  }
  return (double)t.ms;
}
// Every stage reads -1 (did not run) again: called where a training or an encode / decode call starts, so that a
// context that is used again never reports a stage time of an earlier call.
inline void timers_reset(yttm_ctx *c) {
  for (auto &kv : c->timers) { kv.second.ms = -1.f; kv.second.pending = false; }
}
inline uint64_t pow2ceil(uint64_t x) { uint64_t p = 1; while (p < x) p <<= 1; return p; }
// The library's environment knobs (DESIGN §7.5).  env_int: `dflt` when `name` is unset, else its integer value clamped
// to [lo, hi].  A knob is read where it takes effect: the geometry knobs (yttm_geometry_knobs) once per context, the
// others on every call.
inline bool env_set(const char *name) { return std::getenv(name) != nullptr; }
inline int env_int(const char *name, int dflt, int lo, int hi) {
  const char *e = std::getenv(name);
  return e ? std::min(hi, std::max(lo, std::atoi(e))) : dflt;
}
}  // namespace ytc
