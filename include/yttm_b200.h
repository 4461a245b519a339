/* yttm_b200.h — the drop-in boundary: a C ABI over the two BPE hot paths on one H100.
 *
 * The reference (VKCOM/YouTokenToMe) has no FFI of its own; its boundary is the C++ header
 * youtokentome/cpp/bpe.h (train_bpe :19, class BaseEncoder :22-82) bound by Cython
 * (youtokentome/cpp/yttm.pyx:10-49).  This header is what a maintainer binds instead of the
 * bodies of learn_bpe_from_string (bpe.cpp:859-1293) and encode_parallel (bpe.cpp:1697-1738):
 * plain pointers and sizes, int return codes (0 = ok), message via yttm_last_error().
 *
 * Conventions: the caller owns every host buffer; the library owns device memory inside the
 * context.  A context is bound to one CUDA device and is NOT thread-safe (one per host thread).
 * All entry points fail (non-zero) — they never fall back to a CPU path — when CUDA is missing.
 */
#ifndef YTTM_B200_H
#define YTTM_B200_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct yttm_ctx yttm_ctx;
typedef struct yttm_enc yttm_enc;

/* ---- context ------------------------------------------------------------------------------ */
int yttm_ctx_create(int device, yttm_ctx **out);
void yttm_ctx_destroy(yttm_ctx *ctx);
const char *yttm_last_error(const yttm_ctx *ctx); /* ctx may be NULL: error of the last failed create */
int yttm_device_count(void);

/* cudaEvent milliseconds of the last call of the named stage ("char_hist", "word_count",
 * "tokenise", "pair_hist", "merge_loop", "encode", "h2d", "d2h", "enc_spans", "enc_subwords", "decode", "dec_count",
 * "dec_scan", "dec_emit", "dec_e2e"); < 0 if unknown or if the stage did not run in the current training (since the last
 * yttm_train_load_corpus) or the last encode / decode call.  Counters of the last yttm_train_run under the same name:
 * "loop_iters", "loop_refreshes", "loop_launches", "loop_resident", "table_capacity", and "xq_round" (exchange rounds
 * of the merge loop since the context was created or joined a job; they run on across trainings).  Counters of the
 * current training: "feed_pieces" (pieces of a fed corpus, 0 after load_corpus) and "dev_peak_bytes" (the largest sum
 * of the context's device buffers, sampled after every fed piece and every phase). */
double yttm_stage_ms(const yttm_ctx *ctx, const char *stage);
/* number of kernel launches issued by this context so far (bench.py: gpu_launches) */
uint64_t yttm_launch_count(const yttm_ctx *ctx);

/* ---- training: replaces learn_bpe_from_string phases 1-4 (bpe.cpp:859-1293) --------------- */

/* Phase 0 — corpus shard.  `bytes` is a HOST pointer (copied H2D) unless on_device != 0, in
 * which case it is a device pointer that must stay valid until yttm_train_build returns.
 * Replaces fast_read_file_utf8's buffer (bpe.cpp:67-84) as the input of the passes below.
 * Host corpora of >= 64 MB are copied in pieces that end behind an ASCII space / newline; phase 1
 * and the word table of phase 2 run per piece on a second stream behind the copy of the next piece
 * (the calls below then only collect the results; YTTM_TRAIN_PIPELINE=0 turns this off).
 * A context may train again: this call drops whatever an earlier corpus built (words, pair table), so that export_words,
 * dump_pairs, scan_once and run fail until yttm_train_build has run on the new corpus. */
int yttm_train_load_corpus(yttm_ctx *ctx, const char *bytes, uint64_t n, int on_device);

/* Phase 0 for corpora larger than the device's memory: the text is FED in host blocks of any size and boundaries
 * (mid-word and mid-UTF-8 sequence included) between feed_begin and feed_end, instead of one load_corpus.  The library
 * cuts the text into pieces behind a whitespace byte (space, \t .. \r), runs phase 1 and the word split per piece,
 * and merges each piece's distinct words into one device table whose bytes live in a word arena; the corpus itself is
 * never resident.  feed_begin starts a new training like load_corpus; feed copies the caller's bytes before it
 * returns; feed_end returns what yttm_train_char_hist returns, and the arena of unique words becomes the context's
 * text.  char_hist, set_alphabet and build then keep their meaning (build takes the fed words as they are), and so do
 * export_words, dump_pairs, scan_once, run and yttm_train_dist_export_words.  YTTM_TRAIN_FEED_PIECE_KB sets the piece
 * size (read by feed_begin).  feed before feed_begin, and char_hist or build between feed_begin and feed_end, fail. */
int yttm_train_feed_begin(yttm_ctx *ctx);
int yttm_train_feed(yttm_ctx *ctx, const char *bytes, uint64_t n);
int yttm_train_feed_end(yttm_ctx *ctx, uint64_t *data_len, uint64_t *n_distinct);

/* Phase 1 — compute_char_count (bpe.cpp:839-857): *data_len = number of decode units (spaces
 * and invalid bytes included); histogram of valid non-space code points.  *n_distinct = number
 * of code points with a non-zero count. */
int yttm_train_char_hist(yttm_ctx *ctx, uint64_t *data_len, uint64_t *n_distinct);
/* Copies the histogram, ascending code point; both arrays hold n_distinct entries. */
int yttm_train_get_char_hist(yttm_ctx *ctx, uint32_t *cps, uint64_t *counts);
/* Multi-GPU: device pointer to the dense histogram, uint64[*n_u64] with slot [0x110000] =
 * data_len, to be sum-allreduced across ranks by the caller (NCCL) before get_char_hist. */
int yttm_train_char_hist_devptr(yttm_ctx *ctx, void **dptr, uint64_t *n_u64);
/* After an in-place allreduce of that buffer: refresh data_len / n_distinct from it. */
int yttm_train_char_hist_refresh(yttm_ctx *ctx, uint64_t *data_len, uint64_t *n_distinct);

/* Alphabet chosen on the host (compute_alphabet_helper bpe.cpp:316-355, the one floating-point
 * compare of training stays on the host): kept code points and their INTERNAL ids; every other
 * code point is "removed" (remove_rare_chars bpe.cpp:357-380).  space_id = id of U+2581. */
int yttm_train_set_alphabet(yttm_ctx *ctx, const uint32_t *cps, const uint32_t *ids, uint64_t n_kept,
                            uint32_t space_id);

typedef struct yttm_train_stats {
  uint64_t n_bytes;        /* B  corpus bytes on this rank                      */
  uint64_t n_words;        /* W  word occurrences                                */
  uint64_t n_unique;       /* U  unique words (non-empty after char removal)     */
  uint64_t n_tokens;       /* T  tokens of the unique words (sum len + 1)        */
  uint64_t n_pairs;        /* P0 distinct pairs in the initial table             */
  uint64_t table_capacity; /*    slots of the pair table                         */
} yttm_train_stats;

/* Phases 2-3 — compute_word_count (bpe.cpp:388-418) + build_linked_list (bpe.cpp:436-478):
 * word split, dedup with counts, tokenise ([space_id] + char ids), packed uint32 token buffer
 * + offsets + uint64 frequencies, initial pair->count table. */
int yttm_train_build(yttm_ctx *ctx, yttm_train_stats *stats);

/* Multi-GPU word exchange (round 1, kept for callers that gather through the host): export this rank's unique
 * words (tokens, offsets[n_unique+1], freq) to host buffers, or import a concatenation of all ranks' exports and
 * rebuild the pair table from it (duplicates across ranks are harmless: statistics are additive).
 * Preconditions of an imported word set, which words built by the trainer always meet:
 *   - the first token of a word appears at no other position of any word (the role of U+2581: the STREAMING merge
 *     loop relies on it, a pair never straddles two tiles);
 *   - token ids and first_new_id + max_merges of the following yttm_train_run stay below 2^22;
 *   - freq[i] x (tokens of word i) < 2^43: a count change travels through the merge loop as a signed 44-bit value
 *     (checked: import_words fails otherwise).  Pair counts themselves are 64-bit. */
int yttm_train_export_words(yttm_ctx *ctx, uint32_t *tokens, uint64_t tokens_cap, uint32_t *offsets,
                            uint64_t *freq, uint64_t words_cap, uint64_t *n_words, uint64_t *n_tokens);
int yttm_train_import_words(yttm_ctx *ctx, const uint32_t *tokens, uint64_t n_tokens, const uint32_t *offsets,
                            const uint64_t *freq, uint64_t n_words, yttm_train_stats *stats);

/* ---- multi-GPU training: one process (or host thread) per GPU, world <= 8 ------------------------------------
 * Replaces the cooperation of the reference's training threads: the thread partition of the unique words
 * (bpe.cpp:1066-1069), the merge of the per-thread word maps (:1029-1039) and the per-merge exchange of pair counts
 * between workers and main (:789-804, :1099-1108, :1239-1266).  Protocol, every rank in lockstep:
 *   yttm_train_dist_init(ctx, rank, world, handle)   allocate this rank's exchange buffer, get its 128-byte handle
 *   <all-gather the handles, any transport>           (torch.distributed in youtokentome_b200/distributed.py)
 *   yttm_train_dist_connect(ctx, handles)             map every peer's buffer (CUDA IPC; same process: peer access)
 *   load_corpus(shard) / char_hist / <allreduce of the histogram> / set_alphabet      as on one GPU
 *   yttm_train_dist_word_table                        word split + dedup of the shard
 *   yttm_train_dist_export_words                      unique words grouped by owner rank = hash(bytes) % world
 *   <all-to-all of the three device buffers>
 *   yttm_train_dist_import_words                      dedup across ranks (equal words met on one rank), tokenise,
 *                                                     pair table = sum over ranks (exchange rounds through the peers'
 *                                                     buffers, no collective library involved)
 *   yttm_train_run                                    the merge loop: every rank rewrites its own words and stores the
 *                                                     count changes of a merge straight into every peer's exchange
 *                                                     buffer over NVLink; every rank keeps the full table and elects
 *                                                     the same pair.  All ranks return the same rules.
 * A rank whose peer stays silent for YTTM_XQ_TIMEOUT_MS (default 30 000) aborts its kernel instead of hanging. */
int yttm_train_dist_init(yttm_ctx *ctx, uint32_t rank, uint32_t world, void *handle_out /* 128 bytes */);
int yttm_train_dist_connect(yttm_ctx *ctx, const void *handles /* world x 128 bytes, by rank */);
int yttm_train_dist_word_table(yttm_ctx *ctx, uint64_t *n_unique);
/* bytes_per_dst / words_per_dst: world entries each.  *d_bytes: the words of destination 0, 1, ... back to back, each
 * followed by one space; *d_pos (uint64 per word): its first byte relative to its destination's first byte;
 * *d_freq (uint64 per word): its count.  Device memory owned by the context, valid until the next call on it. */
int yttm_train_dist_export_words(yttm_ctx *ctx, uint64_t *bytes_per_dst, uint64_t *words_per_dst, void **d_bytes,
                                 void **d_pos, void **d_freq);
/* the same three buffers after the all-to-all (DEVICE pointers, sources back to back) + the per-source sizes */
int yttm_train_dist_import_words(yttm_ctx *ctx, const void *d_bytes, const uint64_t *bytes_per_src, const void *d_pos,
                                 const void *d_freq, const uint64_t *words_per_src, yttm_train_stats *stats);

/* Phase 4 — the merge loop (main bpe.cpp:1121-1282 + worker_doing_merge :601-811): up to
 * max_merges iterations of { argmax under MergeCandidate::operator< (bpe.cpp:110-126); apply
 * x y -> z over every word; update pair counts }.  New ids are first_new_id, first_new_id+1, ...
 * rules_xyz receives 3 uint32 per merge, freqs the count of the merged pair at merge time.
 * *n_done < max_merges means no pair was left ("WARNING merged only", bpe.cpp:1139). */
int yttm_train_run(yttm_ctx *ctx, uint32_t first_new_id, uint32_t max_merges, uint32_t *rules_xyz,
                   uint64_t *freqs, uint32_t *n_done);

/* Diagnostics for parity tests: copy the live pair table (key = x<<32|y, count > 0). */
int yttm_train_dump_pairs(yttm_ctx *ctx, uint64_t *keys, uint64_t *counts, uint64_t cap, uint64_t *n);

/* One full pair-count scan over the current packed token buffer into a scratch table (the
 * headline "BPE-train scan" kernel; build/rebuild run the same kernel).  Returns its cudaEvent
 * milliseconds and the algorithmic bytes it read (4T + 12U, SURVEY.md §8d). */
int yttm_train_scan_once(yttm_ctx *ctx, double *ms, uint64_t *algo_bytes);

/* Synthetic packed words generated ON DEVICE for roofline measurement of the scan kernel:
 * n_words words of `len` tokens: the first token of word w is 4 + w % n_first (word-initial ids,
 * never used elsewhere - the role of U+2581), the others 4 + n_first + (LCG % (alphabet & 0xffffff));
 * n_first = 1 << (alphabet >> 24).  New ids must start at 4 + n_first + (alphabet & 0xffffff). */
int yttm_train_synth_words(yttm_ctx *ctx, uint64_t n_words, uint32_t len, uint32_t alphabet, uint64_t seed);

/* ---- encoding: replaces encode_parallel / encode_sentence (bpe.cpp:1455-1632, 1697-1738) -- */

/* Model tables (BaseEncoder::fill_from_state bpe.cpp:1667-1690): char2id pairs and rules with
 * FINAL ids as stored in the model file (utils.cpp:50-91). */
int yttm_enc_create(yttm_ctx *ctx, const uint32_t *char_cp, const uint32_t *char_id, uint64_t n_chars,
                    const uint32_t *rules_xyz, uint64_t n_rules, int unk_id, int pad_id, int bos_id, int eos_id,
                    yttm_enc **out);
void yttm_enc_destroy(yttm_enc *enc);

/* encode_as_ids (bpe.cpp:1740): sentence i = bytes[offsets[i], offsets[i+1]).  HOST buffers;
 * H2D / D2H inside.  out_offsets has n_sent+1 entries; *out_n = total ids.  If out_cap is too
 * small returns 2 with *out_n = required size (nothing written).  dropout > 0 draws from
 * Philox4x32-10 keyed (seed, first_sentence_index + i, word byte offset, draw#); the word byte offset is the
 * offset inside the sentence of the first byte of the word's maximal run of non-space units, invalid bytes
 * included ("\xc0\xafabc" is one word at offset 0). */
int yttm_enc_run(yttm_enc *enc, const char *bytes, const uint64_t *offsets, uint64_t n_sent, int bos, int eos,
                 int reverse, double dropout, uint64_t seed, uint64_t first_sentence_index, int32_t *out_ids,
                 uint64_t out_cap, uint64_t *out_offsets, uint64_t *out_n);

/* Same with DEVICE-resident input (d_bytes, d_offsets) and results left on the device:
 * *d_out_ids / *d_out_offsets point into library-owned memory valid until the next call.  The ids are reserved before
 * they are counted, at n_bytes + (1 + bos + eos) * n_sent ids of 4 bytes (the most a batch can produce). */
int yttm_enc_run_device(yttm_enc *enc, const char *d_bytes, const uint64_t *d_offsets, uint64_t n_bytes,
                        uint64_t n_sent, int bos, int eos, int reverse, double dropout, uint64_t seed,
                        uint64_t first_sentence_index, const int32_t **d_out_ids, const uint64_t **d_out_offsets,
                        uint64_t *out_n);

/* ---- source spans and subword pieces of an encode ---------------------------------------------------------------
 * Same batches, arguments, checks and ids as yttm_enc_run / yttm_enc_run_device, plus the bytes every id came from.
 * Span of id j = (spans[2j], spans[2j+1]) = [start, end) in the coordinates of offsets (sentence i is
 * [offsets[i], offsets[i+1]) of them, also for the device forms whose d_bytes is the first byte of sentence 0):
 *   an ordinary id covers a run of valid units (code points, or invalid bytes) of its word: from the first byte of its
 *   first valid unit to the end of its last; an invalid unit between two of its units lies inside, any other in no span;
 *   <UNK> covers its maximal run of out-of-alphabet units the same way; a word-initial U+2581 no rule merged covers no
 *   unit: its span is empty and sits where the next id's span starts; <BOS> = [offsets[i], offsets[i]), <EOS> =
 *   [offsets[i+1], offsets[i+1]); with reverse the (id, span) pairs are reversed together.
 * The first spans / subwords call of an encoder builds its piece table (host work + one upload). */
int yttm_enc_run_spans(yttm_enc *enc, const char *bytes, const uint64_t *offsets, uint64_t n_sent, int bos, int eos,
                       int reverse, double dropout, uint64_t seed, uint64_t first_sentence_index, int32_t *out_ids,
                       uint64_t out_cap, uint64_t *out_offsets, uint64_t *out_spans /* 2 * out_cap */, uint64_t *out_n);
/* *d_out_* point into library-owned memory, complete when the call returns and valid until the next encode call.  The
 * ids and spans are reserved before they are counted, at n_bytes + (1 + bos + eos) * n_sent ids: 20 bytes per id
 * (about 2.6 GB for 128 MB of input), so split batches that do not fit the device at that bound. */
int yttm_enc_run_spans_device(yttm_enc *enc, const char *d_bytes, const uint64_t *d_offsets, uint64_t n_bytes,
                              uint64_t n_sent, int bos, int eos, int reverse, double dropout, uint64_t seed,
                              uint64_t first_sentence_index, const int32_t **d_out_ids, const uint64_t **d_out_offsets,
                              const uint64_t **d_out_spans, uint64_t *out_n);
/* ---- padded rows of an encode ----------------------------------------------------------------------------------
 * Same batches, arguments, checks and dropout stream as yttm_enc_run; sentence i becomes row i of an n_sent x width
 * matrix (row i = ids[i * width, (i + 1) * width)).  With c_i = the ids yttm_enc_run gives sentence i with
 * bos = eos = reverse = 0 and K = width - bos - eos:
 *   row_i = [<BOS>]? + c_i[:K] + [<EOS>]?   (truncation drops ids from the end of the content; <BOS> / <EOS> stay),
 *   reversed as a whole after the truncation with reverse;  lengths[i] = len(row_i);  cells [lengths[i], width) hold
 *   pad_id.  With spans, a kept id has the span yttm_enc_run_spans gives it and a pad cell the empty span
 *   [offsets[i+1], offsets[i+1]) (spans[2 (i width + j)], spans[2 (i width + j) + 1] for cell j of row i).
 * Only the n_sent x width cells are reserved on the device (20 bytes per cell with spans), never the packed bound; a
 * request that does not fit fails with an error.  HOST buffers: width >= max(1, bos + eos) and below 2^31; out_ids holds
 * n_sent * width ids, out_lengths n_sent values, out_spans (NULL = not asked for) 2 * n_sent * width values.  The
 * batch runs in chunks whose rows are copied straight to their place. */
int yttm_enc_run_padded(yttm_enc *enc, const char *bytes, const uint64_t *offsets, uint64_t n_sent, int bos, int eos,
                        int reverse, double dropout, uint64_t seed, uint64_t first_sentence_index, uint64_t width,
                        int32_t pad_id, int32_t *out_ids /* n_sent * width */, uint64_t *out_lengths /* n_sent */,
                        uint64_t *out_spans /* NULL or 2 * n_sent * width */);
/* DEVICE-resident input; width = 0 takes the longest row of the batch, max_i(|c_i| + bos + eos) (0 when every row is
 * empty), at the cost of one counting pass and one 8-byte read-back; *out_width = the width used.  *d_ids /
 * *d_lengths / *d_spans (with_spans, else NULL) point into library-owned memory, complete when the call returns and
 * valid until the next encode call. */
int yttm_enc_run_padded_device(yttm_enc *enc, const char *d_bytes, const uint64_t *d_offsets, uint64_t n_bytes,
                               uint64_t n_sent, int bos, int eos, int reverse, double dropout, uint64_t seed,
                               uint64_t first_sentence_index, uint64_t width /* 0 = longest */, int32_t pad_id,
                               int with_spans, const int32_t **d_ids, const uint64_t **d_lengths,
                               const uint64_t **d_spans, uint32_t *out_width);
/* encode_as_subwords (bpe.cpp:1757) of a batch: one piece per id, piece k = pieces[piece_offsets[k],
 * piece_offsets[k+1]) (UTF-8): the recipe of an ordinary id with its leading U+2581 kept, "<BOS>" / "<EOS>", and for
 * <UNK> the characters of its run (its span's bytes without invalid units).  The pieces of sentence i are
 * [sent_offsets[i], sent_offsets[i+1]).  piece_offsets has *n_pieces + 1 entries, sent_offsets n_sent + 1.  Returns 2
 * with *n_pieces / *n_piece_bytes = the sizes needed when pieces_cap or bytes_cap is too small (nothing written). */
int yttm_enc_run_subwords(yttm_enc *enc, const char *bytes, const uint64_t *offsets, uint64_t n_sent, int bos, int eos,
                          int reverse, double dropout, uint64_t seed, uint64_t first_sentence_index, uint8_t *out_pieces,
                          uint64_t bytes_cap, uint64_t *out_piece_offsets /* pieces_cap + 1 */, uint64_t pieces_cap,
                          uint64_t *out_sent_offsets, uint64_t *n_pieces, uint64_t *n_piece_bytes);
int yttm_enc_run_subwords_device(yttm_enc *enc, const char *d_bytes, const uint64_t *d_offsets, uint64_t n_bytes,
                                 uint64_t n_sent, int bos, int eos, int reverse, double dropout, uint64_t seed,
                                 uint64_t first_sentence_index, const uint8_t **d_pieces, const uint64_t **d_piece_offsets,
                                 const uint64_t **d_sent_offsets, uint64_t *n_pieces, uint64_t *n_piece_bytes);

/* ---- decoding: BaseEncoder::decode (bpe.cpp:1843-1861 + id_to_subword :1774-1807) of a batch ---- */

/* Sentence i = ids[offsets[i], offsets[i+1]) (absolute indices; offsets[0] need not be 0, offsets must not decrease).
 * Ids listed in ignore[n_ignore] (a HOST array) are skipped; any other id outside [0, vocab_size) fails with the
 * host decode's text ("id must be in the range ...") for the first such id in batch order, and nothing is written.
 * Every other id gives its piece (special tokens as "<UNK>" / "<PAD>" / "<BOS>" / "<EOS>", a leading U+2581 as one
 * space); a sentence's text is its pieces back to back without the leading space of its first piece.  Text i =
 * out[out_offsets[i], out_offsets[i+1]), out_offsets has n_sent+1 entries, *out_n = total bytes.  The first call on an
 * encoder builds its piece table (host work + one upload).  At most 2^32 - 16 ids and sentences per call.
 * HOST buffers; returns 2 with *out_n = the size needed when out_cap is too small (nothing written). */
int yttm_dec_run(yttm_enc *enc, const int32_t *ids, const uint64_t *offsets, uint64_t n_sent, const int32_t *ignore,
                 uint64_t n_ignore, uint8_t *out, uint64_t out_cap, uint64_t *out_offsets, uint64_t *out_n);

/* Same with DEVICE-resident ids[n_ids] and offsets; offsets past n_ids are an error.  *d_out / *d_out_offsets point into
 * library-owned memory, complete when the call returns and valid until the next yttm_dec_run_device call on the
 * encoder (yttm_dec_run and the encode calls use other memory, so the ids yttm_enc_run_device returned can be decoded
 * in place). */
int yttm_dec_run_device(yttm_enc *enc, const int32_t *d_ids, uint64_t n_ids, const uint64_t *d_offsets, uint64_t n_sent,
                        const int32_t *ignore, uint64_t n_ignore, const uint8_t **d_out, const uint64_t **d_out_offsets,
                        uint64_t *out_n);

#ifdef __cplusplus
}
#endif
#endif /* YTTM_B200_H */
