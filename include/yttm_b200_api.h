/* yttm_b200_api.h — flat C entry points over the host C++ surface (bpe_b200.h), bound by the
 * Python package with ctypes.  They replace the reference's Cython class
 * (youtokentome/cpp/yttm.pyx:52-181): same operations, same error texts (returned through
 * yttm_api_last_error instead of a C++ Status).  `handle` is an opened model.
 */
#ifndef YTTM_B200_API_H
#define YTTM_B200_API_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

const char *yttm_api_last_error(void *handle); /* handle may be NULL: thread-local error */

/* yttm.pyx:64-85 BPE.train -> train_bpe (bpe.h:19) */
int yttm_api_train(const char *data_path, const char *model_path, int vocab_size, double coverage, int n_threads,
                   int pad_id, int unk_id, int bos_id, int eos_id);
/* learn_bpe_from_string (bpe.cpp:859) on an in-memory corpus; model_path may be "" */
int yttm_api_train_memory(const char *text, uint64_t n, const char *model_path, int vocab_size, double coverage,
                          int pad_id, int unk_id, int bos_id, int eos_id);
/* count_words (bpe_b200.h): the word-count table of the text of in_fd (a file or a pipe; in_fd < 0: text[n]), also
 * written as TSV to tsv_path when it is not NULL ("-" = stdout).  sizes[4] = unique words, their bytes, separators,
 * data_len.  0 ok, 1 error.  yttm_api_result_words then copies the table, sorted by count descending and bytes
 * ascending, of this thread's last count_words: bytes[sizes[1]], offsets[sizes[0] + 1], counts[sizes[0]]. */
int yttm_api_count_words(int in_fd, const char *text, uint64_t n, const char *tsv_path, uint64_t *sizes);
void yttm_api_result_words(uint8_t *bytes, uint64_t *offsets, uint64_t *counts);
/* train_counts (bpe_b200.h): trains from a word-count table, the arrays of yttm_train_feed_words (on_device != 0:
 * device memory; separators UINT64_MAX: one per occurrence) or, when tsv_path is not NULL, a TSV file as count_words
 * writes it.  The model and the errors are train_bpe's on any text with the same words, counts and separators. */
int yttm_api_train_counts(const uint8_t *bytes, const uint64_t *offsets, const uint64_t *counts, uint64_t n,
                          uint64_t separators, int on_device, const char *tsv_path, const char *model_path,
                          int vocab_size, double coverage, int n_threads, int pad_id, int unk_id, int bos_id,
                          int eos_id);
/* sizes and stage times of the last training on this thread (see TrainReport); returns #values */
int yttm_api_train_report(double *out, int n);
/* frees the device buffers train_bpe keeps cached for the calling thread (vkcom::release_training_cache) */
void yttm_api_release_training_cache(void);
/* training contexts currently cached by all threads of the process (vkcom::training_cache_held) */
int yttm_api_training_cache_held(void);

/* yttm.pyx:58-62 BPE.__init__ -> BaseEncoder(model_path, n_threads, &status) */
void *yttm_api_open(const char *model_path, int n_threads);
void yttm_api_close(void *handle);
int yttm_api_vocab_size(void *handle);
void yttm_api_set_dropout_seed(void *handle, uint64_t seed);

/* Thread safety: every call that runs kernels holds a per-handle mutex; results of the two-call entry points below
 * (encode_ids -> result_ids, encode_subwords / decode / vocab / id_to_subword -> result_counts / _text / _offsets) are
 * kept per CALLING THREAD, so threads sharing one handle never see each other's results. */

/* yttm.pyx:87-107 encode(output_type='id'): sentence i = bytes[offsets[i], offsets[i+1]) */
int yttm_api_encode_ids(void *handle, const char *bytes, const uint64_t *offsets, uint64_t n_sent, int bos, int eos,
                        int reverse, double dropout, uint64_t *total_ids);
void yttm_api_result_ids(void *handle, int32_t *ids, uint64_t *offsets /* n_sent + 1 */);
/* the same in ONE call into caller-owned buffers: 0 ok, 1 error, 2 ids_cap too small (*total_ids = size needed);
 * ids_cap >= bytes + 3 * n_sent always suffices */
int yttm_api_encode_ids_into(void *handle, const char *bytes, const uint64_t *offsets, uint64_t n_sent, int bos, int eos,
                             int reverse, double dropout, int32_t *ids_out, uint64_t ids_cap, uint64_t *offsets_out,
                             uint64_t *total_ids);
/* device-resident input and output (pointers into library-owned device memory, valid until the next encode call) */
int yttm_api_encode_device(void *handle, const char *d_bytes, const uint64_t *d_offsets, uint64_t n_bytes, uint64_t n_sent,
                           int bos, int eos, int reverse, double dropout, const int32_t **d_ids,
                           const uint64_t **d_id_offsets, uint64_t *total_ids);

/* yttm.pyx:108-124 encode(output_type='subword').  Piece lists are LENGTH-FRAMED (a piece may hold any character):
 * the call returns the byte length of all pieces (or -1); yttm_api_result_counts gives (pieces, sentences),
 * yttm_api_result_text the bytes, yttm_api_result_offsets the byte offset of every piece (+ end, n_pieces + 1 values)
 * and the first piece of every sentence (+ end, n_sentences + 1 values; may be NULL). */
int64_t yttm_api_encode_subwords(void *handle, const char *bytes, const uint64_t *offsets, uint64_t n_sent, int bos,
                                 int eos, int reverse, double dropout);
void yttm_api_result_counts(void *handle, uint64_t *n_pieces, uint64_t *n_sentences);
void yttm_api_result_text(void *handle, char *out);
void yttm_api_result_offsets(void *handle, uint64_t *piece_off, uint64_t *sent_off);

/* encode with the source span of every id (yttm_enc_run_spans of yttm_b200.h): spans_out holds 2 * ids_cap values,
 * (start, end) per id in the coordinates of offsets; 0 ok, 1 error, 2 ids_cap too small (*total_ids = size needed) */
int yttm_api_encode_spans_into(void *handle, const char *bytes, const uint64_t *offsets, uint64_t n_sent, int bos, int eos,
                               int reverse, double dropout, int32_t *ids_out, uint64_t ids_cap, uint64_t *offsets_out,
                               uint64_t *spans_out, uint64_t *total_ids);
int yttm_api_encode_spans_device(void *handle, const char *d_bytes, const uint64_t *d_offsets, uint64_t n_bytes,
                                 uint64_t n_sent, int bos, int eos, int reverse, double dropout, const int32_t **d_ids,
                                 const uint64_t **d_id_offsets, const uint64_t **d_spans, uint64_t *total_ids);
/* encode as padded rows (yttm_enc_run_padded of yttm_b200.h): ids_out holds n_sent * width ids, lengths_out n_sent
 * values, spans_out (may be NULL) 2 * n_sent * width; pad_id = YTTM_PAD_FROM_MODEL takes the model's pad id (an error
 * if the model has none), any other value must fit in int32.  The device form takes width = 0 for the longest row and
 * sets *out_width; its results are library-owned device memory valid until the next encode call.  0 ok, 1 error. */
#define YTTM_PAD_FROM_MODEL INT64_MIN
int yttm_api_encode_padded_into(void *handle, const char *bytes, const uint64_t *offsets, uint64_t n_sent, int bos, int eos,
                                int reverse, double dropout, uint64_t width, int64_t pad_id, int32_t *ids_out,
                                uint64_t *lengths_out, uint64_t *spans_out);
int yttm_api_encode_padded_device(void *handle, const char *d_bytes, const uint64_t *d_offsets, uint64_t n_bytes,
                                  uint64_t n_sent, int bos, int eos, int reverse, double dropout, uint64_t width,
                                  int64_t pad_id, int with_spans, const int32_t **d_ids, const uint64_t **d_lengths,
                                  const uint64_t **d_spans, uint32_t *out_width);
/* encode as overlapping windows (yttm_enc_run_windows_device of yttm_b200.h): *n_rows rows of width ids, stride content
 * ids of overlap between the windows of a sentence, and per row its length, sentence and start; pad_id as for the padded
 * rows.  Results are library-owned device memory valid until the next encode call.  0 ok, 1 error. */
int yttm_api_encode_windows_device(void *handle, const char *d_bytes, const uint64_t *d_offsets, uint64_t n_bytes,
                                   uint64_t n_sent, int bos, int eos, int reverse, double dropout, uint64_t width,
                                   uint64_t stride, int64_t pad_id, int with_spans, const int32_t **d_ids,
                                   const uint64_t **d_lengths, const uint64_t **d_sentence, const uint64_t **d_start,
                                   const uint64_t **d_spans, uint64_t *n_rows);
/* encode(output_type='subword') on the GPU (yttm_enc_run_subwords): the same pieces as yttm_api_encode_subwords, into
 * caller-owned buffers; 0 ok, 1 error, 2 a capacity too small (*n_pieces / *n_bytes = sizes needed) */
int yttm_api_encode_subwords_into(void *handle, const char *bytes, const uint64_t *offsets, uint64_t n_sent, int bos,
                                  int eos, int reverse, double dropout, uint8_t *pieces, uint64_t bytes_cap,
                                  uint64_t *piece_offsets /* pieces_cap + 1 */, uint64_t pieces_cap,
                                  uint64_t *sent_offsets /* n_sent + 1 */, uint64_t *n_pieces, uint64_t *n_bytes);
int yttm_api_encode_subwords_device(void *handle, const char *d_bytes, const uint64_t *d_offsets, uint64_t n_bytes,
                                    uint64_t n_sent, int bos, int eos, int reverse, double dropout, const uint8_t **d_pieces,
                                    const uint64_t **d_piece_offsets, const uint64_t **d_sent_offsets, uint64_t *n_pieces,
                                    uint64_t *n_piece_bytes);

/* yttm.pyx:136-158 decode: one piece per sentence; id_to_subword: one piece; vocab: vocab_size pieces */
int64_t yttm_api_decode(void *handle, const int32_t *ids, const uint64_t *offsets, uint64_t n_sent,
                        const int32_t *ignore, uint64_t n_ignore);
/* decode on the GPU (yttm_dec_run of yttm_b200.h): text i = text[text_offsets[i], text_offsets[i+1]); 0 ok, 1 error,
 * 2 text_cap too small (*total_bytes = size needed, nothing written) */
int yttm_api_decode_into(void *handle, const int32_t *ids, const uint64_t *offsets, uint64_t n_sent,
                         const int32_t *ignore, uint64_t n_ignore, uint8_t *text, uint64_t text_cap,
                         uint64_t *text_offsets, uint64_t *total_bytes);
/* device-resident ids / offsets and results (pointers into library-owned device memory, valid until the next
 * decode_device call; not the memory of yttm_api_encode_device's results) */
int yttm_api_decode_device(void *handle, const int32_t *d_ids, uint64_t n_ids, const uint64_t *d_offsets,
                           uint64_t n_sent, const int32_t *ignore, uint64_t n_ignore, const uint8_t **d_text,
                           const uint64_t **d_text_offsets, uint64_t *total_bytes);
int64_t yttm_api_id_to_subword(void *handle, int id);
int yttm_api_subword_to_id(void *handle, const char *subword);
int64_t yttm_api_vocab(void *handle);

int yttm_api_encode_cli(void *handle, const char *output_type, int stream, int bos, int eos, int reverse,
                        double dropout);
int yttm_api_decode_cli(void *handle, const int32_t *ignore, uint64_t n_ignore);
/* BaseEncoder::encode_file: the lines of in_fd to <out_path>.ids.npy + <out_path>.offsets.npy, or with text != 0 to
 * out_path ("-" = stdout) as `yttm encode --output_type id` writes them; uses the handle's dropout seed and counter.
 * stats[3] = lines, ids, input bytes.  0 ok, 1 error. */
int yttm_api_encode_file(void *handle, int in_fd, const char *out_path, int text, int bos, int eos, int reverse,
                         double dropout, uint64_t *stats);
/* BaseEncoder::encode_file_subwords: the lines of in_fd to out_path ("-" = stdout) as `yttm encode --output_type
 * subword` writes them; uses the handle's dropout seed and counter.  stats[3] = lines, pieces, input bytes.  0 ok,
 * 1 error. */
int yttm_api_encode_file_subwords(void *handle, int in_fd, const char *out_path, int bos, int eos, int reverse,
                                  double dropout, uint64_t *stats);
/* BaseEncoder::decode_file: with text != 0 the id text of in_fd, else the pair <in_prefix>.ids.npy +
 * <in_prefix>.offsets.npy, decoded to out_path ("-" = stdout) as `yttm decode` prints it; ignore[n_ignore] as for
 * decode.  stats[3] = lines, ids, text bytes written.  0 ok, 1 error. */
int yttm_api_decode_file(void *handle, int in_fd, const char *in_prefix, const char *out_path, int text,
                         const int32_t *ignore, uint64_t n_ignore, uint64_t *stats);
void yttm_api_vocab_cli(void *handle, int verbose);

/* order of the char2id lines of a model file written by the reference (BPEState::dump, utils.cpp:57-59):
 * filled[n] = code points by ascending id -> out[n].  Host only, needs no GPU. */
int yttm_api_dump_order(const uint32_t *filled, uint64_t n, uint32_t *out);
/* BPEState::load (utils.cpp:68-91) then BPEState::dump (utils.cpp:50-66) of a model file: rewrites any valid
 * model file in the reference's canonical line order.  Host only.  0 = ok, 1 = cannot read in_path. */
int yttm_api_redump(const char *in_path, const char *out_path);

/* raw yttm_ctx* / yttm_enc* of an opened model, for callers of yttm_b200.h */
void *yttm_api_device_context(void *handle);
void *yttm_api_device_encoder(void *handle);

#ifdef __cplusplus
}
#endif
#endif
