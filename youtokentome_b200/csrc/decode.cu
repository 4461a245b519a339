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

// NL: every sentence is followed by one '\n' (the decode stream's lines)
template <bool NL>
__device__ __forceinline__ void dec_count(DecArgs a) {
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
    if (lane == 0) a.sent_bytes[s] = sum + (NL ? 1 : 0);
  }
}

__global__ void __launch_bounds__(256) dec_count_kernel(DecArgs a) { dec_count<false>(a); }
__global__ void __launch_bounds__(256) dec_count_nl_kernel(DecArgs a) { dec_count<true>(a); }

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

template <bool NL>
__device__ __forceinline__ void dec_emit(DecArgs a, const unsigned long long *__restrict__ out_off,
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
    if (NL && lane == 0) out[pos] = '\n';  // a byte store: no round wrote a full word over it
  }
}

__global__ void __launch_bounds__(256) dec_emit_kernel(DecArgs a, const unsigned long long *__restrict__ out_off,
                                                       uint8_t *__restrict__ out) {
  dec_emit<false>(a, out_off, out);
}
__global__ void __launch_bounds__(256) dec_emit_nl_kernel(DecArgs a, const unsigned long long *__restrict__ out_off,
                                                          uint8_t *__restrict__ out) {
  dec_emit<true>(a, out_off, out);
}

// ---- the decode stream's kernels ----

__global__ void __launch_bounds__(256) widen_ids_kernel(const uint16_t *__restrict__ in, uint64_t n,
                                                        int32_t *__restrict__ out) {
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) out[i] = in[i];
}

// Id text: the ids of a line are what `std::stringstream >> int` reads from it (BaseEncoder::decode of a string):
// tokens [+-]?[0-9]+ between whitespace (' ', \t, \v, \f, \r; the line's '\n' counts as whitespace) or right after the
// previous token, read until the first stop: a byte that is neither whitespace, a digit nor a sign, a sign not followed by
// a digit, or a token outside int32.  Every digit run before the first stop is a token, so a line's ids are its digit
// runs that end before the first stop, and each is decided by bytes near its last digit: its value is its last 10
// digits, unless a nonzero digit lies before them (found with a scan of the last byte that is not '0').  A warp reads
// a line in rounds of 512 bytes (16 per lane, one 16-byte load); nothing walks a line byte by byte.
constexpr uint32_t IDT_ROUND = 512;

// bit k: byte q + k of the line [lo, hi) is a digit / a sign / another stop byte / not '0' (bytes outside the line are
// whitespace, and not '0')
__device__ __forceinline__ void id_text_classes(const uint8_t *__restrict__ p, uint64_t n, uint64_t q, uint64_t lo,
                                                uint64_t hi, uint32_t *dig, uint32_t *sign, uint32_t *other,
                                                uint32_t *nz) {
  uint32_t w[4] = {0x0a0a0a0au, 0x0a0a0a0au, 0x0a0a0a0au, 0x0a0a0a0au};
  if (q + 16 <= n) {
    const uint4 v = __ldg(reinterpret_cast<const uint4 *>(p + q));
    w[0] = v.x; w[1] = v.y; w[2] = v.z; w[3] = v.w;
  } else {
    for (uint32_t k = 0; k < 16 && q + k < n; k++)
      w[k >> 2] = (w[k >> 2] & ~(0xffu << (8 * (k & 3)))) | ((uint32_t)p[q + k] << (8 * (k & 3)));
  }
  uint32_t d = 0, s = 0, o = 0, z = 0;
#pragma unroll
  for (uint32_t k = 0; k < 16; k++) {
    const uint32_t x = (w[k >> 2] >> (8 * (k & 3))) & 0xffu;
    const bool isd = x - '0' < 10u, iss = x == '+' || x == '-', isw = x == ' ' || x - 9u < 5u;
    d |= (uint32_t)isd << k;
    s |= (uint32_t)iss << k;
    o |= (uint32_t)(!isd && !iss && !isw) << k;
    z |= (uint32_t)(x != '0') << k;
  }
  const uint32_t a = q < lo ? (uint32_t)(lo - q) : 0u, b = q + 16 <= hi ? 16u : hi > q ? (uint32_t)(hi - q) : 0u;
  const uint32_t in = a < b ? ((1u << b) - 1u) & ~((1u << a) - 1u) : 0u;
  *dig = d & in;
  *sign = s & in;
  *other = o & in;
  *nz = (z | ~in) & 0xffffu;
}

// A lane's view of the last byte that is not '0': its chunk (q, z), the chunk before (zprev) and the scan values in
// front of each
struct NzWin {
  int64_t q, excl, exclprev;
  uint32_t z, zprev;
};

// the position of the last byte at or before x that is not '0' (x >= q - 16)
__device__ __forceinline__ int64_t last_nonzero(const NzWin &w, int64_t x) {
  if (x >= w.q) {
    const uint32_t m = w.z & (0xffffu >> (15 - (uint32_t)(x - w.q)));
    return m ? w.q + 31 - __clz((int)m) : w.excl;
  }
  const uint32_t m = w.zprev & (0xffffu >> (15 - (uint32_t)(x - w.q + 16)));
  return m ? w.q - 16 + 31 - __clz((int)m) : w.exclprev;
}

// The token whose last digit is byte e of the line starting at lo: false when its value is outside int32.
__device__ __forceinline__ bool token_value(const uint8_t *__restrict__ p, int64_t lo, int64_t e, const NzWin &w,
                                            int32_t *out) {
  uint64_t v = 0, mul = 1;
  int64_t nd = 0;
  for (; nd < 10 && e - nd >= lo; nd++) {
    const uint32_t x = (uint32_t)__ldg(p + e - nd) - '0';
    if (x >= 10u) break;
    v += x * mul;
    mul *= 10;
  }
  int64_t before = e - nd;  // the byte in front of the digits read
  if (nd == 10 && before >= lo && (uint32_t)__ldg(p + before) - '0' < 10u) {  // a longer run: leading zeros or overflow
    before = last_nonzero(w, before);
    if (before >= lo && (uint32_t)__ldg(p + before) - '0' < 10u) return false;
  }
  const bool neg = before >= lo && __ldg(p + before) == '-';
  if (v > (neg ? 2147483648ull : 2147483647ull)) return false;
  *out = (int32_t)(neg ? 0u - (uint32_t)v : (uint32_t)v);
  return true;
}

// The ids of the line [lo, hi) of the n bytes at p: their number (every lane); WRITE: to out[0 ..].
template <bool WRITE>
__device__ __forceinline__ uint64_t id_text_line(const uint8_t *__restrict__ p, uint64_t n, uint64_t lo, uint64_t hi,
                                                 unsigned lane, int32_t *__restrict__ out) {
  uint64_t count = 0;
  int64_t carry_incl = (int64_t)lo - 1, carry_excl = (int64_t)lo - 1;  // the scan in front of the line: its boundary
  uint32_t carry_z = 0xffffu;
  for (uint64_t r = lo & ~15ull; r < hi; r += IDT_ROUND) {  // warp-uniform
    const uint64_t q = r + 16 * lane;
    uint32_t D, S, O, Z;
    id_text_classes(p, n, q, lo, hi, &D, &S, &O, &Z);
    uint32_t dn = __shfl_down_sync(0xffffffffu, D, 1) & 1u;  // the byte behind the chunk is a digit
    if (lane == 31) dn = q + 16 < hi && (uint32_t)__ldg(p + q + 16) - '0' < 10u;
    const uint32_t Dnext = (D >> 1) | (dn << 15);
    const uint32_t E = D & ~Dnext, stop = O | (S & ~Dnext);  // last digits of tokens; stop bytes
    int64_t incl = (int64_t)q + 31 - __clz((int)Z);  // Z has bits for the bytes outside the line: never 0 past it
    if (!Z) incl = -1;
    if (lane == 0) incl = max(incl, carry_incl);
#pragma unroll
    for (unsigned o = 1; o < 32; o <<= 1) {
      const int64_t y = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl = max(incl, y);
    }
    NzWin w;
    w.q = (int64_t)q;
    w.z = Z;
    w.excl = __shfl_up_sync(0xffffffffu, incl, 1);
    w.zprev = __shfl_up_sync(0xffffffffu, Z, 1);
    if (lane == 0) { w.excl = carry_incl; w.zprev = carry_z; }
    w.exclprev = __shfl_up_sync(0xffffffffu, w.excl, 1);
    if (lane == 0) w.exclprev = carry_excl;
    uint32_t ov = 0;
    for (uint32_t m = E; m; m &= m - 1) {
      const int k = __ffs((int)m) - 1;
      int32_t v;
      if (!token_value(p, (int64_t)lo, (int64_t)q + k, w, &v)) ov |= 1u << k;
    }
    const uint32_t kill = stop | ov;
    const unsigned bk = __ballot_sync(0xffffffffu, kill != 0);
    uint32_t keep = E;
    if (bk) {
      const unsigned first = (unsigned)__ffs((int)bk) - 1;
      if (lane > first) keep = 0;
      else if (lane == first) keep &= (1u << (__ffs((int)kill) - 1)) - 1u;
    }
    const uint32_t cnt = (uint32_t)__popc(keep);
    uint32_t before = cnt;
#pragma unroll
    for (unsigned o = 1; o < 32; o <<= 1) {
      const uint32_t y = __shfl_up_sync(0xffffffffu, before, o);
      if (lane >= o) before += y;
    }
    if (WRITE) {
      int32_t *dst = out + count + before - cnt;
      for (uint32_t m = keep; m; m &= m - 1) {
        int32_t v = 0;
        token_value(p, (int64_t)lo, (int64_t)q + (__ffs((int)m) - 1), w, &v);
        *dst++ = v;
      }
    }
    count += __shfl_sync(0xffffffffu, before, 31);
    if (bk) break;
    carry_incl = __shfl_sync(0xffffffffu, incl, 31);
    carry_excl = __shfl_sync(0xffffffffu, w.excl, 31);
    carry_z = __shfl_sync(0xffffffffu, Z, 31);
  }
  return count;
}

// warp per line (offs: n_lines + 1 byte offsets of the lines): the number of its ids
__global__ void __launch_bounds__(256) id_text_count_kernel(const uint8_t *__restrict__ p, uint64_t n,
                                                            const unsigned long long *__restrict__ offs, uint64_t n_lines,
                                                            unsigned long long *__restrict__ line_ids) {
  const unsigned lane = threadIdx.x & 31;
  const uint64_t warp = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const uint64_t nwarps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
  for (uint64_t s = warp; s < n_lines; s += nwarps) {
    const uint64_t c = id_text_line<false>(p, n, offs[s], offs[s + 1], lane, nullptr);
    if (lane == 0) line_ids[s] = c;
  }
}

// warp per line: its ids at ids[id_off[s] ..]
__global__ void __launch_bounds__(256) id_text_write_kernel(const uint8_t *__restrict__ p, uint64_t n,
                                                            const unsigned long long *__restrict__ offs, uint64_t n_lines,
                                                            const unsigned long long *__restrict__ id_off,
                                                            int32_t *__restrict__ ids) {
  const unsigned lane = threadIdx.x & 31;
  const uint64_t warp = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const uint64_t nwarps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
  for (uint64_t s = warp; s < n_lines; s += nwarps) id_text_line<true>(p, n, offs[s], offs[s + 1], lane, ids + id_off[s]);
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
// to out / out_off (n_sent + 1 offsets).  The bytes are only written when *total <= out_cap.  nl: every sentence's text
// is followed by one '\n'.
int dec_device(yttm_enc *e, const int32_t *d_ids, uint64_t id_base, uint64_t id_lim, const uint64_t *d_offs,
               uint64_t n_sent, const int32_t *ignore, uint64_t n_ignore, ytc::DevBuf *out, ytc::DevBuf *out_off_buf,
               uint64_t out_cap, uint64_t *total, bool nl = false) {
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
  if (nl) dec_count_nl_kernel<<<(unsigned)sblocks, 256, 0, c->stream>>>(a);
  else dec_count_kernel<<<(unsigned)sblocks, 256, 0, c->stream>>>(a);
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
    if (nl) dec_emit_nl_kernel<<<(unsigned)sblocks, 256, 0, c->stream>>>(a, out_off, out->as<uint8_t>());
    else dec_emit_kernel<<<(unsigned)sblocks, 256, 0, c->stream>>>(a, out_off, out->as<uint8_t>());
    ytc::timer_end(c, "dec_emit");
    c->launches++;
  }
  ytc::timer_end(c, "decode");
  YT_CUDA(c, cudaGetLastError());
  return 0;
}

}  // namespace

// =====================================================================================================================
// Decode stream (yttm_dec_stream_*): ids or id text fed in blocks runs through the shared piece pipeline of the encode
// stream (yttm_piece_pipe), and each piece runs on the device as
//   YTTM_STREAM_IDS16   widen_ids_kernel: the 16-bit ids copied in become int32
//   YTTM_STREAM_TEXT    the line split of the encode stream (yttm_line_split), then
//                       id_text_count_kernel   warp per line: the number of its ids
//                       scan                   the lines' id offsets + the piece's ids (one 8-byte read-back)
//                       id_text_write_kernel   warp per line: its ids
//   dec_device, nl      the text of every line and its '\n' (dec_count_nl_kernel / scan / dec_emit_nl_kernel)
//   add_base_kernel     line ends as global byte counts
struct yttm_dec_stream {
  yttm_enc *e = nullptr;
  int format = YTTM_STREAM_IDS32;
  std::vector<int32_t> ignore;
  yttm_piece_pipe pipe;
  ytc::DevBuf in[2], out[2], out_off[2];  // per slot: the piece copied in; its text and line offsets
  ytc::DevBuf wide, tiles, offs, line_ids, id_off, ids;  // per piece (the pieces' kernels run in order on one stream)
  uint64_t lines = 0, ids_out = 0, bytes = 0;
};

void yttm_dec_stream_free(yttm_dec_stream *s) {
  if (!s) return;
  yttm_pipe_free(&s->pipe);
  ytc::DevBuf *b[] = {&s->in[0], &s->in[1], &s->out[0], &s->out[1], &s->out_off[0], &s->out_off[1], &s->wide, &s->tiles,
                      &s->offs, &s->line_ids, &s->id_off, &s->ids};
  for (auto *x : b) x->release();
  s->e->dec_stream = nullptr;
  delete s;
}

namespace {

// "dec_stream_dev_peak_bytes": the decode tables and buffers of the encoder and the stream's, sampled after each piece
void note_dec_stream_peak(yttm_dec_stream *S) {
  yttm_dec *d = S->e->dec;
  uint64_t sum = 0;
  ytc::DevBuf *b[] = {&d->table, &d->ign, &d->sent_bytes, &d->ctl, &S->in[0], &S->in[1], &S->out[0], &S->out[1],
                      &S->out_off[0], &S->out_off[1], &S->wide, &S->tiles, &S->offs, &S->line_ids, &S->id_off, &S->ids};
  for (auto *x : b) sum += x->cap;
  S->e->ctx->dec_stream_peak = std::max(S->e->ctx->dec_stream_peak, (double)sum);
}

// The kernels of the piece in slot s (yttm_piece_pipe::run).
int dec_stream_run(void *owner, int s, const void **out_data, const unsigned long long **out_ends) {
  yttm_dec_stream *S = static_cast<yttm_dec_stream *>(owner);
  yttm_enc *e = S->e;
  yttm_ctx *c = e->ctx;
  yttm_piece_pipe::Piece &P = S->pipe.pc[s];
  const uint8_t *d = S->in[s].as<uint8_t>();
  const int32_t *ids = nullptr;
  const uint64_t *offs = nullptr;
  uint64_t id_base = 0, id_lim = 0;
  if (S->format == YTTM_STREAM_TEXT) {
    if (yttm_line_split(c, d, P.n_bytes, P.open_end, &S->tiles, &S->offs, &P.n_lines)) return 1;
    YT_CUDA(c, S->line_ids.reserve((P.n_lines + 1) * 8));
    unsigned long long *lc = S->line_ids.as<unsigned long long>(), *lo = S->offs.as<unsigned long long>();
    ytc::timer_begin(c, "dec_stream_parse");
    const unsigned blocks = (unsigned)std::max<uint64_t>(std::min<uint64_t>((P.n_lines + 7) / 8, (uint64_t)c->n_sm * 8), 1);
    id_text_count_kernel<<<blocks, 256, 0, c->stream>>>(d, P.n_bytes, lo, P.n_lines, lc);
    c->launches++;
    YT_CUDA(c, S->id_off.reserve((P.n_lines + 1) * 8));
    unsigned long long *id_off = S->id_off.as<unsigned long long>();
    if (yttm_device_scan_u64(c, lc, P.n_lines, id_off, id_off + P.n_lines)) return 1;
    unsigned long long n_ids = 0;
    YT_CUDA(c, cudaMemcpyAsync(&n_ids, id_off + P.n_lines, 8, cudaMemcpyDeviceToHost, c->stream));
    YT_CUDA(c, cudaStreamSynchronize(c->stream));
    YT_CUDA(c, S->ids.reserve(n_ids * 4 + 16));
    id_text_write_kernel<<<blocks, 256, 0, c->stream>>>(d, P.n_bytes, lo, P.n_lines, id_off, S->ids.as<int32_t>());
    c->launches++;
    ytc::timer_end(c, "dec_stream_parse");
    ids = S->ids.as<int32_t>();
    offs = reinterpret_cast<const uint64_t *>(id_off);
    id_lim = n_ids;
  } else {
    // the piece: its ids, then its line ends as global id counts (yttm_piece_pipe)
    const uint64_t n_ids = P.n_bytes / S->pipe.unit;
    offs = reinterpret_cast<const uint64_t *>(d + ((P.n_bytes + 15) & ~15ull));
    id_base = P.first_id;
    id_lim = id_base + n_ids;
    ids = reinterpret_cast<const int32_t *>(d);
    if (S->format == YTTM_STREAM_IDS16) {
      YT_CUDA(c, S->wide.reserve(n_ids * 4 + 16));
      const unsigned blocks = (unsigned)std::max<uint64_t>(std::min<uint64_t>((n_ids + 255) / 256, (uint64_t)c->n_sm * 8), 1);
      widen_ids_kernel<<<blocks, 256, 0, c->stream>>>(reinterpret_cast<const uint16_t *>(d), n_ids, S->wide.as<int32_t>());
      c->launches++;
      ids = S->wide.as<int32_t>();
    }
  }
  uint64_t total = 0;
  if (dec_device(e, ids, id_base, id_lim, offs, P.n_lines, S->ignore.data(), S->ignore.size(), &S->out[s], &S->out_off[s],
                 ~0ull, &total, true))
    return 1;
  unsigned long long *ends = S->out_off[s].as<unsigned long long>() + 1;
  if (S->bytes) yttm_add_base(c, ends, P.n_lines, (unsigned long long)S->bytes);
  *out_data = S->out[s].p;
  *out_ends = ends;
  P.n_out = total;
  S->lines += P.n_lines;
  S->ids_out += id_lim - id_base;
  S->bytes += total;
  c->dec_stream_pieces += 1;
  note_dec_stream_peak(S);
  return 0;
}

// a failed stream call: the stream is closed, the error kept
int dec_stream_failed(yttm_enc *e) {
  const std::string err = e->ctx->err;
  yttm_dec_stream_free(e->dec_stream);
  cudaGetLastError();
  e->ctx->err = err;
  return 1;
}

// the stream of a feed / end call, or 1 with the error recorded
int dec_stream_of(yttm_enc *e, const char *who, int text) {
  if (!e) return yttm_enc_check(e, who, 0, 0);
  if (!e->dec_stream) YT_FAIL(e->ctx, std::string(who) + ": yttm_dec_stream_begin has not run");
  if (text >= 0 && (e->dec_stream->format == YTTM_STREAM_TEXT) != (text != 0)) {
    e->ctx->err = std::string(who) + (text ? ": the stream takes ids (yttm_dec_stream_feed_ids)"
                                           : ": the stream takes id text (yttm_dec_stream_feed)");
    return dec_stream_failed(e);
  }
  return 0;
}

}  // namespace

extern "C" {

int yttm_dec_stream_begin(yttm_enc *e, int format, const int32_t *ignore, uint64_t n_ignore, yttm_enc_sink sink,
                          void *user) {
  if (yttm_enc_check(e, "yttm_dec_stream_begin", 0, 0)) return 1;
  yttm_ctx *c = e->ctx;
  if (format != YTTM_STREAM_IDS16 && format != YTTM_STREAM_IDS32 && format != YTTM_STREAM_TEXT)
    YT_FAIL(c, "yttm_dec_stream_begin: format must be YTTM_STREAM_IDS16, YTTM_STREAM_IDS32 or YTTM_STREAM_TEXT");
  if (!sink) YT_FAIL(c, "yttm_dec_stream_begin: no sink");
  if (yttm_pipe_init(e)) return 1;
  if (!e->dec) e->dec = new yttm_dec();
  yttm_dec_stream *S = new yttm_dec_stream();
  S->e = e;
  S->format = format;
  S->ignore.assign(ignore, ignore + n_ignore);
  yttm_piece_pipe &p = S->pipe;
  p.e = e;
  p.piece = (uint64_t)ytc::env_int("YTTM_DEC_STREAM_PIECE_KB", 32 << 10, 1, INT_MAX) << 10;
  p.unit = format == YTTM_STREAM_TEXT ? 0 : format == YTTM_STREAM_IDS16 ? 2 : 4;
  p.dev_in[0] = &S->in[0];
  p.dev_in[1] = &S->in[1];
  p.run = dec_stream_run;
  p.owner = S;
  p.sink = sink;
  p.user = user;
  p.who = "yttm_dec_stream";
  e->dec_stream = S;
  c->dec_stream_pieces = 0;
  c->dec_stream_peak = 0;
  return 0;
}

int yttm_dec_stream_feed(yttm_enc *e, const char *bytes, uint64_t n) {
  if (dec_stream_of(e, "yttm_dec_stream_feed", 1)) return 1;
  return yttm_pipe_feed_text(&e->dec_stream->pipe, bytes, n) ? dec_stream_failed(e) : 0;
}

int yttm_dec_stream_feed_ids(yttm_enc *e, const void *ids, uint64_t n_ids, const uint64_t *line_ends, uint64_t n_lines) {
  if (dec_stream_of(e, "yttm_dec_stream_feed_ids", 0)) return 1;
  yttm_piece_pipe &p = e->dec_stream->pipe;
  uint64_t prev = p.ids_in;
  bool ok = true;
  for (uint64_t k = 0; k < n_lines; prev = line_ends[k++]) ok &= line_ends[k] >= prev;
  if (!ok || prev != p.ids_in + n_ids) {
    e->ctx->err = "yttm_dec_stream_feed_ids: line_ends must not decrease, start at the ids fed before (" +
                  std::to_string(p.ids_in) + ") and end at those plus n_ids";
    return dec_stream_failed(e);
  }
  return yttm_pipe_feed_lines(&p, ids, n_ids, line_ends, n_lines) ? dec_stream_failed(e) : 0;
}

int yttm_dec_stream_end(yttm_enc *e, uint64_t *n_lines, uint64_t *n_ids, uint64_t *n_bytes) {
  if (dec_stream_of(e, "yttm_dec_stream_end", -1)) return 1;
  if (yttm_pipe_end(&e->dec_stream->pipe)) return dec_stream_failed(e);
  if (n_lines) *n_lines = e->dec_stream->lines;
  if (n_ids) *n_ids = e->dec_stream->ids_out;
  if (n_bytes) *n_bytes = e->dec_stream->bytes;
  yttm_dec_stream_free(e->dec_stream);
  return 0;
}

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
