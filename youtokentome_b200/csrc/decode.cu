// decode.cu — batch decode (ids -> UTF-8 text) on one H100, behind yttm_dec_run* of include/yttm_b200.h.
//
// Computes BaseEncoder::decode (bpe_host.cpp; the reference's bpe.cpp:1843-1861 + id_to_subword :1774-1807) for a
// packed batch: per sentence, ids in ignore_ids are skipped (before validation), any other id outside [0, V) is an
// error, every kept id contributes its piece (special tokens "<UNK>" ...; otherwise the UTF-8 of its recipe with a
// leading U+2581 turned into one ASCII space), and the leading space of the FIRST kept piece is dropped.
//   piece table           built on the host from the model tables on the first decode call of an encoder, one upload:
//                         piece_off u32[V+1] into piece_bytes (16-byte padded) + a V-bit "starts with a space" map
//   dec_count_kernel      warp per sentence: byte count of the sentence's text; invalid ids -> atomicMin of their
//                         position, malformed offsets -> error flag
//   scan                  exclusive scan of the byte counts (yttm_device_scan_u64) -> u64 output offsets + total;
//                         one D2H of (total, first bad id, offsets flag), the only host round trip of a call
//   dec_emit_kernel       warp per sentence, 32 ids per round: a warp scan places the round's pieces, then the lanes
//                         write the round's bytes as aligned 32-bit words, each byte's piece found by a shuffle search
//                         over the 32 places (a long piece is spread over the lanes); the partial words at both ends
//                         of a round may share their word with the neighbouring sentence and are stored byte by byte
#include <algorithm>
#include <cstring>
#include <string>

#include "common.cuh"
#include "enc_state.cuh"

using namespace yt;

namespace {

constexpr uint32_t MAX_PIECE = 1u << 27;  // bytes of one piece: 32 of them sum to less than 2^32 (u32 warp scan)

struct DecArgs {
  const int32_t *ids;          // id at absolute index j is ids[j - id_base]
  uint64_t id_base, id_lim;    // offsets must lie in [id_base, id_lim]
  const uint64_t *offs;        // n_sent + 1, absolute, non-decreasing
  uint64_t n_sent;
  const uint32_t *piece_off;   // V + 1
  const uint32_t *lead;        // V bits: the piece starts with ' ' (a leading U+2581)
  const uint8_t *bytes;        // piece bytes
  uint32_t vocab;
  const uint32_t *ign;         // V-bit ignore map, nullptr = nothing ignored
  const int32_t *ign_extra;    // ignored values outside [0, V), ascending
  uint32_t n_extra;
  unsigned long long *sent_bytes;  // per sentence
  unsigned long long *ctl;         // [0] total (scan), [1] first invalid id position (~0 = none), [2] offsets flag
};

__device__ __forceinline__ bool bit_of(const uint32_t *m, uint32_t i) { return (m[i >> 5] >> (i & 31)) & 1u; }

__device__ __forceinline__ bool in_extra(const DecArgs &a, int32_t v) {
  uint32_t lo = 0, hi = a.n_extra;
  while (lo < hi) {
    const uint32_t mid = (lo + hi) >> 1;
    const int32_t x = a.ign_extra[mid];
    if (x == v) return true;
    if (x < v) lo = mid + 1; else hi = mid;
  }
  return false;
}

// the sentence range [lo, hi) of sentence s, false if its offsets are malformed (warp-uniform)
__device__ __forceinline__ bool sent_range(const DecArgs &a, uint64_t s, uint64_t *lo, uint64_t *hi) {
  *lo = a.offs[s];
  *hi = a.offs[s + 1];
  return *lo >= a.id_base && *lo <= *hi && *hi <= a.id_lim;
}

// one id of a round: kept (not ignored and valid) -> its piece; *bad = invalid and not ignored
__device__ __forceinline__ bool look(const DecArgs &a, int32_t id, uint32_t *src, uint32_t *len, bool *bad) {
  *bad = false;
  if ((uint32_t)id < a.vocab) {
    if (a.ign && bit_of(a.ign, (uint32_t)id)) return false;
    *src = __ldg(a.piece_off + id);
    *len = __ldg(a.piece_off + id + 1) - *src;
    return true;
  }
  *bad = !in_extra(a, id);
  return false;
}

__global__ void __launch_bounds__(256) dec_count_kernel(DecArgs a) {
  const unsigned lane = threadIdx.x & 31;
  const uint64_t warp = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const uint64_t nwarps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
  for (uint64_t s = warp; s < a.n_sent; s += nwarps) {
    uint64_t lo, hi;
    if (!sent_range(a, s, &lo, &hi)) {  // warp-uniform
      if (lane == 0) { a.ctl[2] = 1; a.sent_bytes[s] = 0; }
      continue;
    }
    unsigned long long sum = 0;
    bool first = true;  // no kept id seen yet
    for (uint64_t j0 = lo; j0 < hi; j0 += 32) {  // warp-uniform
      const uint64_t j = j0 + lane;
      uint32_t src = 0, len = 0;
      bool bad = false, kept = false;
      int32_t id = 0;
      if (j < hi) {
        id = a.ids[j - a.id_base];
        kept = look(a, id, &src, &len, &bad);
      }
      const unsigned b_bad = __ballot_sync(0xffffffffu, bad);
      if (b_bad && lane == (unsigned)__ffs((int)b_bad) - 1) atomicMin(a.ctl + 1, (unsigned long long)j);
      if (first) {
        const unsigned b = __ballot_sync(0xffffffffu, kept);
        if (b) {
          first = false;
          if (lane == (unsigned)__ffs((int)b) - 1 && bit_of(a.lead, (uint32_t)id)) len -= 1;  // the strip
        }
      }
      sum += len;
    }
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    if (lane == 0) a.sent_bytes[s] = sum;
  }
}

// Bytes [0, T) of a round go to out[R0 ..]; lane k holds the inclusive end `incl` of piece k in the round and
// d = (first source byte of piece k) - (its start in the round), so round byte r of piece k is bytes[d + r].
__device__ __forceinline__ void emit_round(const DecArgs &a, uint8_t *__restrict__ out, uint64_t R0, uint32_t T,
                                           uint32_t incl, int64_t d, unsigned lane) {
  const uint64_t w_first = R0 >> 2, w_last = (R0 + T - 1) >> 2;
  for (uint64_t wb = w_first; wb <= w_last; wb += 32) {  // warp-uniform
    const uint64_t w = wb + lane;
    const bool active = w <= w_last;
    uint32_t word = 0, have = 0;
#pragma unroll
    for (int t = 0; t < 4; t++) {
      const int64_t r = (int64_t)(4 * w + t) - (int64_t)R0;
      const bool in = active && r >= 0 && r < (int64_t)T;
      const uint32_t rr = in ? (uint32_t)r : 0u;
      uint32_t k = 0;  // number of pieces that end at or before byte rr = the piece of byte rr
#pragma unroll
      for (uint32_t step = 16; step; step >>= 1)
        if (__shfl_sync(0xffffffffu, incl, k + step - 1) <= rr) k += step;
      const int64_t dk = __shfl_sync(0xffffffffu, d, k);
      if (in) { word |= (uint32_t)__ldg(a.bytes + dk + rr) << (8 * t); have |= 1u << t; }
    }
    if (have == 15u) {
      *reinterpret_cast<uint32_t *>(out + 4 * w) = word;  // inside this round: no other warp writes this word
    } else {
#pragma unroll
      for (int t = 0; t < 4; t++)
        if ((have >> t) & 1u) out[4 * w + t] = (uint8_t)(word >> (8 * t));
    }
  }
}

__global__ void __launch_bounds__(256) dec_emit_kernel(DecArgs a, const unsigned long long *__restrict__ out_off,
                                                       uint8_t *__restrict__ out) {
  const unsigned lane = threadIdx.x & 31;
  const uint64_t warp = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const uint64_t nwarps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
  for (uint64_t s = warp; s < a.n_sent; s += nwarps) {
    uint64_t lo, hi;
    sent_range(a, s, &lo, &hi);  // checked by dec_count_kernel: this kernel runs on valid input only
    uint64_t pos = out_off[s];
    bool first = true;
    for (uint64_t j0 = lo; j0 < hi; j0 += 32) {  // warp-uniform
      const uint64_t j = j0 + lane;
      uint32_t src = 0, len = 0;
      bool bad = false, kept = false;
      int32_t id = 0;
      if (j < hi) {
        id = a.ids[j - a.id_base];
        kept = look(a, id, &src, &len, &bad);
      }
      if (first) {
        const unsigned b = __ballot_sync(0xffffffffu, kept);
        if (b) {
          first = false;
          if (lane == (unsigned)__ffs((int)b) - 1 && bit_of(a.lead, (uint32_t)id)) { src += 1; len -= 1; }
        }
      }
      uint32_t incl = len;
      for (int o = 1; o < 32; o <<= 1) {
        const uint32_t y = __shfl_up_sync(0xffffffffu, incl, o);
        if ((int)lane >= o) incl += y;
      }
      const uint32_t T = __shfl_sync(0xffffffffu, incl, 31);
      if (T) emit_round(a, out, pos, T, incl, (int64_t)src - (int64_t)(incl - len), lane);
      pos += T;
    }
  }
}

void append_utf8(uint32_t x, std::string *out) {  // the host encoder's token2word (bpe_host.cpp)
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

}  // namespace

struct yttm_dec {
  ytc::DevBuf table;  // piece_off | lead bits | piece bytes
  const uint32_t *piece_off = nullptr, *lead = nullptr;
  const uint8_t *bytes = nullptr;
  uint64_t table_bytes = 0;
  // per call; the results of yttm_dec_run_device (out, out_off) outlive the call, so the host-buffer entry point
  // stages its results in buffers of its own (h_out, h_out_off)
  ytc::DevBuf d_ids, d_offs, ign, sent_bytes, ctl, out_off, out, h_out_off, h_out;
  std::vector<uint32_t> h_ign;
  void release() {
    ytc::DevBuf *b[] = {&table, &d_ids, &d_offs, &ign, &sent_bytes, &ctl, &out_off, &out, &h_out_off, &h_out};
    for (auto *x : b) x->release();
  }
};

void yttm_dec_free(yttm_dec *d) {
  if (!d) return;
  d->release();
  delete d;
}

// O(sum of piece bytes) host work.  The recipe of a rule's product is the concatenation of its operands' recipes at the
// time of the rule (fill_from_state), a special id takes its token.
int yttm_model_pieces(yttm_enc *e, const char *who, std::vector<std::string> *raw_out, std::vector<uint8_t> *special_out) {
  yttm_ctx *c = e->ctx;
  const std::string w = who;
  const uint64_t V = e->vocab;
  if (V >= 0x7fffffffull) YT_FAIL(c, w + ": vocabulary too large");
  std::vector<std::string> &raw = *raw_out;
  raw.assign(V, std::string());
  std::vector<uint8_t> have(V, 0);
  for (size_t i = 0; i < e->h_char_cp.size(); i++) {
    const uint32_t id = e->h_char_id[i];
    if (id >= V) YT_FAIL(c, w + ": model has a character id outside [0, vocab_size): " + std::to_string(id));
    raw[id].clear();
    append_utf8(e->h_char_cp[i], &raw[id]);
    have[id] = 1;
  }
  for (size_t i = 0; 3 * i + 2 < e->h_rules_xyz.size(); i++) {
    const uint32_t x = e->h_rules_xyz[3 * i], y = e->h_rules_xyz[3 * i + 1], z = e->h_rules_xyz[3 * i + 2];
    if (x >= V || y >= V || z >= V) YT_FAIL(c, w + ": model has a rule id outside [0, vocab_size): rule " + std::to_string(i));
    if (!have[x] || !have[y]) YT_FAIL(c, w + ": model rule " + std::to_string(i) + " uses an id without a piece");
    if (raw[x].size() + raw[y].size() >= MAX_PIECE) YT_FAIL(c, w + ": model piece of id " + std::to_string(z) + " is over 128 MB");
    std::string r = raw[x] + raw[y];
    raw[z] = std::move(r);
    have[z] = 1;
  }
  std::vector<uint8_t> &special = *special_out;
  special.assign(V, 0);
  const std::pair<int, const char *> sp[] = {{e->unk, "<UNK>"}, {e->pad, "<PAD>"}, {e->bos, "<BOS>"}, {e->eos, "<EOS>"}};
  for (auto &p : sp)
    if (p.first >= 0 && (uint64_t)p.first < V) { raw[p.first] = p.second; have[p.first] = 1; special[p.first] = 1; }
  for (uint64_t i = 0; i < V; i++)
    if (!have[i]) YT_FAIL(c, w + ": model has no piece for id " + std::to_string(i));
  return 0;
}

namespace {

// The decode piece of every id in [0, V) and one upload.
int build_piece_table(yttm_enc *e) {
  yttm_ctx *c = e->ctx;
  const uint64_t V = e->vocab;
  std::vector<std::string> raw;
  std::vector<uint8_t> special;
  if (yttm_model_pieces(e, "decode", &raw, &special)) return 1;
  const uint64_t n_bits = (V + 31) / 32;
  std::vector<uint32_t> off(V + 1), lead(n_bits, 0);
  uint64_t total = 0;
  for (uint64_t i = 0; i < V; i++) {
    if (!special[i] && raw[i].compare(0, 3, "\xe2\x96\x81") == 0) {  // replace_space: a leading U+2581 is one space
      raw[i].replace(0, 3, " ");
      lead[i >> 5] |= 1u << (i & 31);
    }
    off[i] = (uint32_t)total;
    total += raw[i].size();
    if (total > 0xffffff00ull) YT_FAIL(c, "decode: piece table over 4 GB");
  }
  off[V] = (uint32_t)total;
  auto up16 = [](uint64_t x) { return (x + 15) & ~15ull; };
  const uint64_t a_lead = up16((V + 1) * 4), a_bytes = a_lead + up16(n_bits * 4), size = a_bytes + up16(total + 16);
  std::vector<uint8_t> h(size, 0);
  std::memcpy(h.data(), off.data(), (V + 1) * 4);
  std::memcpy(h.data() + a_lead, lead.data(), n_bits * 4);
  for (uint64_t i = 0; i < V; i++) std::memcpy(h.data() + a_bytes + off[i], raw[i].data(), raw[i].size());
  yttm_dec *d = e->dec;
  YT_CUDA(c, d->table.reserve(size));
  YT_CUDA(c, cudaMemcpyAsync(d->table.p, h.data(), size, cudaMemcpyHostToDevice, c->stream));
  YT_CUDA(c, cudaStreamSynchronize(c->stream));
  d->piece_off = d->table.as<uint32_t>();
  d->lead = reinterpret_cast<const uint32_t *>(d->table.as<uint8_t>() + a_lead);
  d->bytes = d->table.as<uint8_t>() + a_bytes;
  d->table_bytes = size;
  return 0;
}

std::string offsets_error(uint64_t n_ids) {
  return "decode: offsets must be non-decreasing and lie within the ids (n_ids = " + std::to_string(n_ids) + ")";
}

// Runs the decode of a batch on the device.  Ids at absolute positions [id_base, id_lim) are d_ids[0 ..]; the results go
// to out / out_off (n_sent + 1 offsets).  The bytes are only written when *total <= out_cap.
int dec_device(yttm_enc *e, const int32_t *d_ids, uint64_t id_base, uint64_t id_lim, const uint64_t *d_offs,
               uint64_t n_sent, const int32_t *ignore, uint64_t n_ignore, ytc::DevBuf *out, ytc::DevBuf *out_off_buf,
               uint64_t out_cap, uint64_t *total) {
  yttm_ctx *c = e->ctx;
  *total = 0;
  if (id_lim - id_base >= 0xfffffff0ull || n_sent >= 0xfffffff0ull)
    YT_FAIL(c, "decode batch too large: at most 2^32 - 16 ids / sentences per call (split the batch)");
  yttm_dec *d = e->dec;
  if (!d->piece_off && build_piece_table(e)) return 1;
  const uint32_t V = (uint32_t)e->vocab;
  YT_CUDA(c, out_off_buf->reserve((n_sent + 2) * 8));
  if (n_sent == 0) {
    YT_CUDA(c, cudaMemsetAsync(out_off_buf->p, 0, 8, c->stream));
    YT_CUDA(c, cudaStreamSynchronize(c->stream));
    return 0;
  }
  DecArgs a;
  a.ids = d_ids; a.id_base = id_base; a.id_lim = id_lim;
  a.offs = d_offs; a.n_sent = n_sent;
  a.piece_off = d->piece_off; a.lead = d->lead; a.bytes = d->bytes; a.vocab = V;
  a.ign = nullptr; a.ign_extra = nullptr; a.n_extra = 0;
  if (n_ignore) {  // V-bit map of the ignored ids in range + the other ignored values, sorted: one upload
    const uint64_t n_bits = (V + 31) / 32;
    std::vector<int32_t> extra;
    d->h_ign.assign(n_bits, 0);
    for (uint64_t i = 0; i < n_ignore; i++) {
      if ((uint32_t)ignore[i] < V) d->h_ign[(uint32_t)ignore[i] >> 5] |= 1u << (ignore[i] & 31);
      else extra.push_back(ignore[i]);
    }
    std::sort(extra.begin(), extra.end());
    for (int32_t v : extra) d->h_ign.push_back((uint32_t)v);
    YT_CUDA(c, d->ign.reserve(d->h_ign.size() * 4));
    YT_CUDA(c, cudaMemcpyAsync(d->ign.p, d->h_ign.data(), d->h_ign.size() * 4, cudaMemcpyHostToDevice, c->stream));
    a.ign = d->ign.as<uint32_t>();
    a.ign_extra = d->ign.as<int32_t>() + n_bits;
    a.n_extra = (uint32_t)extra.size();
  }
  YT_CUDA(c, d->sent_bytes.reserve(n_sent * 8));
  YT_CUDA(c, d->ctl.reserve(32));
  a.sent_bytes = d->sent_bytes.as<unsigned long long>();
  a.ctl = d->ctl.as<unsigned long long>();
  YT_CUDA(c, cudaMemsetAsync(a.ctl, 0, 32, c->stream));
  YT_CUDA(c, cudaMemsetAsync(a.ctl + 1, 0xff, 8, c->stream));
  ytc::timer_begin(c, "decode");
  const uint64_t sblocks = std::max<uint64_t>(std::min<uint64_t>((n_sent + 7) / 8, (uint64_t)c->n_sm * 8), 1);
  ytc::timer_begin(c, "dec_count");
  dec_count_kernel<<<(unsigned)sblocks, 256, 0, c->stream>>>(a);
  ytc::timer_end(c, "dec_count");
  c->launches++;
  unsigned long long *out_off = out_off_buf->as<unsigned long long>();
  ytc::timer_begin(c, "dec_scan");
  if (yttm_device_scan_u64(c, a.sent_bytes, n_sent, out_off, a.ctl)) return 1;
  ytc::timer_end(c, "dec_scan");
  unsigned long long h_ctl[3] = {0, 0, 0};
  YT_CUDA(c, cudaMemcpyAsync(h_ctl, a.ctl, 24, cudaMemcpyDeviceToHost, c->stream));
  YT_CUDA(c, cudaMemcpyAsync(out_off + n_sent, a.ctl, 8, cudaMemcpyDeviceToDevice, c->stream));
  YT_CUDA(c, cudaStreamSynchronize(c->stream));
  if (h_ctl[2]) { ytc::timer_end(c, "decode"); YT_FAIL(c, offsets_error(id_lim)); }
  if (h_ctl[1] != ~0ull) {  // the first invalid id in batch order: read its value (error path only)
    int32_t bad = 0;
    YT_CUDA(c, cudaMemcpy(&bad, d_ids + (h_ctl[1] - id_base), 4, cudaMemcpyDeviceToHost));
    ytc::timer_end(c, "decode");
    YT_FAIL(c, "id must be in the range [0, vocab_size - 1]. Current value: vocab_size = " + std::to_string(V) +
                   "; id=" + std::to_string(bad) + ";");
  }
  *total = h_ctl[0];
  if (h_ctl[0] <= out_cap) {
    YT_CUDA(c, out->reserve(h_ctl[0] + 16));
    ytc::timer_begin(c, "dec_emit");
    dec_emit_kernel<<<(unsigned)sblocks, 256, 0, c->stream>>>(a, out_off, out->as<uint8_t>());
    ytc::timer_end(c, "dec_emit");
    c->launches++;
  }
  ytc::timer_end(c, "decode");
  YT_CUDA(c, cudaGetLastError());
  return 0;
}

}  // namespace

extern "C" {

int yttm_dec_run_device(yttm_enc *e, const int32_t *d_ids, uint64_t n_ids, const uint64_t *d_offsets, uint64_t n_sent,
                        const int32_t *ignore, uint64_t n_ignore, const uint8_t **d_out, const uint64_t **d_out_offsets,
                        uint64_t *out_n) {
  if (yttm_enc_check(e, "yttm_dec_run_device", 0, 0)) return 1;
  yttm_ctx *c = e->ctx;
  if (!e->dec) e->dec = new yttm_dec();
  yttm_dec *d = e->dec;
  if (dec_device(e, d_ids, 0, n_ids, d_offsets, n_sent, ignore, n_ignore, &d->out, &d->out_off, ~0ull, out_n)) return 1;
  YT_CUDA(c, cudaStreamSynchronize(c->stream));  // the results are complete for readers on any stream
  if (d_out) *d_out = d->out.cap ? d->out.as<uint8_t>() : nullptr;
  if (d_out_offsets) *d_out_offsets = d->out_off.as<uint64_t>();
  return 0;
}

int yttm_dec_run(yttm_enc *e, const int32_t *ids, const uint64_t *offsets, uint64_t n_sent, const int32_t *ignore,
                 uint64_t n_ignore, uint8_t *out, uint64_t out_cap, uint64_t *out_offsets, uint64_t *out_n) {
  if (yttm_enc_check(e, "yttm_dec_run", 0, 0)) return 1;
  yttm_ctx *c = e->ctx;
  *out_n = 0;
  const uint64_t base = offsets[0], lim = offsets[n_sent];
  if (lim < base) YT_FAIL(c, offsets_error(lim));
  if (!e->dec) e->dec = new yttm_dec();
  yttm_dec *d = e->dec;
  const uint64_t n = lim - base;
  YT_CUDA(c, d->d_ids.reserve(n * 4 + 16));
  YT_CUDA(c, d->d_offs.reserve((n_sent + 1) * 8));
  ytc::timer_begin(c, "dec_e2e");
  if (n) YT_CUDA(c, cudaMemcpyAsync(d->d_ids.p, ids + base, n * 4, cudaMemcpyHostToDevice, c->stream));
  YT_CUDA(c, cudaMemcpyAsync(d->d_offs.p, offsets, (n_sent + 1) * 8, cudaMemcpyHostToDevice, c->stream));
  uint64_t total = 0;
  if (dec_device(e, d->d_ids.as<int32_t>(), base, lim, d->d_offs.as<uint64_t>(), n_sent, ignore, n_ignore, &d->h_out,
                 &d->h_out_off, out_cap, &total))
    return 1;
  *out_n = total;
  if (total > out_cap) { c->err = "yttm_dec_run: output buffer too small"; return 2; }
  if (total) YT_CUDA(c, cudaMemcpyAsync(out, d->h_out.p, total, cudaMemcpyDeviceToHost, c->stream));
  YT_CUDA(c, cudaMemcpyAsync(out_offsets, d->h_out_off.p, (n_sent + 1) * 8, cudaMemcpyDeviceToHost, c->stream));
  YT_CUDA(c, cudaStreamSynchronize(c->stream));
  ytc::timer_end(c, "dec_e2e");
  return 0;
}

}  // extern "C"
