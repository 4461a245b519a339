"""ctypes binding of libyttm_b200.so (built in-tree by csrc/Makefile).  Plays the role of the
reference's Cython extension module `_youtokentome_cython` (youtokentome/cpp/yttm.pyx).  There
is deliberately no fallback: if the CUDA library is missing, importing the product path fails."""
import ctypes as C
import os
import subprocess

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libyttm_b200.so")


def build(force=False):
    """Compile the CUDA library in-tree (nvcc cross-compiles sm_90a without a GPU)."""
    args = ["make", "-s", "-C", os.path.join(_HERE, "csrc")]
    if force:
        subprocess.run(args + ["clean"], check=True)
    subprocess.run(args + ["all"], check=True)


_lib = None


def lib():
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            "youtokentome_b200: %s is missing - run `python -c 'import __graft_entry__ as g; g.build()'` "
            "(there is no CPU fallback)" % LIB_PATH)
    _lib = bind(C.CDLL(LIB_PATH))
    return _lib


# yttm_enc_sink of include/yttm_b200.h (the sink of both streams): (user, data, n_bytes, line_ends, n_lines) -> 0 or a
# failure
ENC_SINK = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64), C.c_uint64)
STREAM_IDS16, STREAM_IDS32, STREAM_TEXT, STREAM_SUBWORD = 0, 1, 2, 3


def bind(L):
    """Declare the C signatures of include/yttm_b200.h and include/yttm_b200_api.h on a loaded library."""
    vp, cp, u64, i32, dbl, i64 = C.c_void_p, C.c_char_p, C.c_uint64, C.c_int, C.c_double, C.c_int64
    sig = {
        # ---- host-level API (include/yttm_b200_api.h)
        "yttm_api_last_error": (cp, [vp]),
        "yttm_api_train": (i32, [cp, cp, i32, dbl, i32, i32, i32, i32, i32]),
        "yttm_api_train_memory": (i32, [cp, u64, cp, i32, dbl, i32, i32, i32, i32]),
        "yttm_api_train_report": (i32, [vp, i32]),
        "yttm_api_count_words": (i32, [i32, vp, u64, cp, vp]),
        "yttm_api_result_words": (None, [vp, vp, vp]),
        "yttm_api_train_counts": (i32, [vp, vp, vp, u64, u64, i32, cp, cp, i32, dbl, i32, i32, i32, i32, i32]),
        "yttm_api_release_training_cache": (None, []),
        "yttm_api_training_cache_held": (i32, []),
        "yttm_api_open": (vp, [cp, i32]),
        "yttm_api_close": (None, [vp]),
        "yttm_api_vocab_size": (i32, [vp]),
        "yttm_api_set_dropout_seed": (None, [vp, u64]),
        "yttm_api_encode_ids": (i32, [vp, vp, vp, u64, i32, i32, i32, dbl, C.POINTER(u64)]),
        "yttm_api_result_ids": (None, [vp, vp, vp]),
        "yttm_api_encode_ids_into": (i32, [vp, vp, vp, u64, i32, i32, i32, dbl, vp, u64, vp, C.POINTER(u64)]),
        "yttm_api_encode_device": (i32, [vp, vp, vp, u64, u64, i32, i32, i32, dbl, C.POINTER(vp), C.POINTER(vp), C.POINTER(u64)]),
        "yttm_api_result_counts": (None, [vp, C.POINTER(u64), C.POINTER(u64)]),
        "yttm_api_result_offsets": (None, [vp, vp, vp]),
        "yttm_api_encode_subwords": (i64, [vp, vp, vp, u64, i32, i32, i32, dbl]),
        "yttm_api_result_text": (None, [vp, vp]),
        "yttm_api_encode_spans_into": (i32, [vp, vp, vp, u64, i32, i32, i32, dbl, vp, u64, vp, vp, C.POINTER(u64)]),
        "yttm_api_encode_spans_device": (i32, [vp, vp, vp, u64, u64, i32, i32, i32, dbl, C.POINTER(vp), C.POINTER(vp),
                                               C.POINTER(vp), C.POINTER(u64)]),
        "yttm_api_encode_padded_into": (i32, [vp, vp, vp, u64, i32, i32, i32, dbl, u64, i64, vp, vp, vp]),
        "yttm_api_encode_padded_device": (i32, [vp, vp, vp, u64, u64, i32, i32, i32, dbl, u64, i64, i32, C.POINTER(vp),
                                                C.POINTER(vp), C.POINTER(vp), C.POINTER(C.c_uint32)]),
        "yttm_api_encode_windows_device": (i32, [vp, vp, vp, u64, u64, i32, i32, i32, dbl, u64, u64, i64, i32,
                                                 C.POINTER(vp), C.POINTER(vp), C.POINTER(vp), C.POINTER(vp), C.POINTER(vp),
                                                 C.POINTER(u64)]),
        "yttm_api_encode_subwords_into": (i32, [vp, vp, vp, u64, i32, i32, i32, dbl, vp, u64, vp, u64, vp, C.POINTER(u64),
                                                C.POINTER(u64)]),
        "yttm_api_encode_subwords_device": (i32, [vp, vp, vp, u64, u64, i32, i32, i32, dbl, C.POINTER(vp), C.POINTER(vp),
                                                  C.POINTER(vp), C.POINTER(u64), C.POINTER(u64)]),
        "yttm_api_decode": (i64, [vp, vp, vp, u64, vp, u64]),
        "yttm_api_decode_into": (i32, [vp, vp, vp, u64, vp, u64, vp, u64, vp, C.POINTER(u64)]),
        "yttm_api_decode_device": (i32, [vp, vp, u64, vp, u64, vp, u64, C.POINTER(vp), C.POINTER(vp), C.POINTER(u64)]),
        "yttm_api_id_to_subword": (i64, [vp, i32]),
        "yttm_api_subword_to_id": (i32, [vp, cp]),
        "yttm_api_vocab": (i64, [vp]),
        "yttm_api_encode_cli": (i32, [vp, cp, i32, i32, i32, i32, dbl]),
        "yttm_api_decode_cli": (i32, [vp, vp, u64]),
        "yttm_api_encode_file": (i32, [vp, i32, cp, i32, i32, i32, i32, dbl, vp]),
        "yttm_api_encode_file_subwords": (i32, [vp, i32, cp, i32, i32, i32, dbl, vp]),
        "yttm_api_decode_file": (i32, [vp, i32, cp, cp, i32, vp, u64, vp]),
        "yttm_api_vocab_cli": (None, [vp, i32]),
        "yttm_api_dump_order": (i32, [vp, u64, vp]),
        "yttm_api_redump": (i32, [cp, cp]),
        "yttm_api_device_context": (vp, [vp]),
        "yttm_api_device_encoder": (vp, [vp]),
        # ---- device ABI (include/yttm_b200.h)
        "yttm_device_count": (i32, []),
        "yttm_ctx_create": (i32, [i32, C.POINTER(vp)]),
        "yttm_ctx_destroy": (None, [vp]),
        "yttm_last_error": (cp, [vp]),
        "yttm_stage_ms": (dbl, [vp, cp]),
        "yttm_launch_count": (u64, [vp]),
        "yttm_train_load_corpus": (i32, [vp, vp, u64, i32]),
        "yttm_train_feed_begin": (i32, [vp]),
        "yttm_train_feed": (i32, [vp, vp, u64]),
        "yttm_train_feed_end": (i32, [vp, C.POINTER(u64), C.POINTER(u64)]),
        "yttm_train_feed_words": (i32, [vp, vp, vp, vp, u64, u64, i32]),
        "yttm_train_fed_words": (i32, [vp, vp, u64, vp, vp, u64, C.POINTER(u64), C.POINTER(u64), C.POINTER(u64)]),
        "yttm_train_char_hist": (i32, [vp, C.POINTER(u64), C.POINTER(u64)]),
        "yttm_train_get_char_hist": (i32, [vp, vp, vp]),
        "yttm_train_char_hist_devptr": (i32, [vp, C.POINTER(vp), C.POINTER(u64)]),
        "yttm_train_char_hist_refresh": (i32, [vp, C.POINTER(u64), C.POINTER(u64)]),
        "yttm_train_set_alphabet": (i32, [vp, vp, vp, u64, C.c_uint32]),
        "yttm_train_build": (i32, [vp, vp]),
        "yttm_train_export_words": (i32, [vp, vp, u64, vp, vp, u64, C.POINTER(u64), C.POINTER(u64)]),
        "yttm_train_import_words": (i32, [vp, vp, u64, vp, vp, u64, vp]),
        "yttm_train_dist_init": (i32, [vp, C.c_uint32, C.c_uint32, vp]),
        "yttm_train_dist_connect": (i32, [vp, vp]),
        "yttm_train_dist_word_table": (i32, [vp, C.POINTER(u64)]),
        "yttm_train_dist_export_words": (i32, [vp, vp, vp, C.POINTER(vp), C.POINTER(vp), C.POINTER(vp)]),
        "yttm_train_dist_import_words": (i32, [vp, vp, vp, vp, vp, vp, vp]),
        "yttm_train_run": (i32, [vp, C.c_uint32, C.c_uint32, vp, vp, C.POINTER(C.c_uint32)]),
        "yttm_train_dump_pairs": (i32, [vp, vp, vp, u64, C.POINTER(u64)]),
        "yttm_train_scan_once": (i32, [vp, C.POINTER(dbl), C.POINTER(u64)]),
        "yttm_train_synth_words": (i32, [vp, u64, C.c_uint32, C.c_uint32, u64]),
        "yttm_enc_create": (i32, [vp, vp, vp, u64, vp, u64, i32, i32, i32, i32, C.POINTER(vp)]),
        "yttm_enc_destroy": (None, [vp]),
        "yttm_enc_run": (i32, [vp, vp, vp, u64, i32, i32, i32, dbl, u64, u64, vp, u64, vp, C.POINTER(u64)]),
        "yttm_enc_run_device": (i32, [vp, vp, vp, u64, u64, i32, i32, i32, dbl, u64, u64, C.POINTER(vp), C.POINTER(vp),
                                      C.POINTER(u64)]),
        "yttm_enc_run_spans": (i32, [vp, vp, vp, u64, i32, i32, i32, dbl, u64, u64, vp, u64, vp, vp, C.POINTER(u64)]),
        "yttm_enc_run_spans_device": (i32, [vp, vp, vp, u64, u64, i32, i32, i32, dbl, u64, u64, C.POINTER(vp),
                                            C.POINTER(vp), C.POINTER(vp), C.POINTER(u64)]),
        "yttm_enc_run_padded": (i32, [vp, vp, vp, u64, i32, i32, i32, dbl, u64, u64, u64, C.c_int32, vp, vp, vp]),
        "yttm_enc_run_padded_device": (i32, [vp, vp, vp, u64, u64, i32, i32, i32, dbl, u64, u64, u64, C.c_int32, i32,
                                             C.POINTER(vp), C.POINTER(vp), C.POINTER(vp), C.POINTER(C.c_uint32)]),
        "yttm_enc_run_windows_device": (i32, [vp, vp, vp, u64, u64, i32, i32, i32, dbl, u64, u64, u64, u64, C.c_int32,
                                              i32, C.POINTER(vp), C.POINTER(vp), C.POINTER(vp), C.POINTER(vp),
                                              C.POINTER(vp), C.POINTER(u64)]),
        "yttm_enc_run_subwords": (i32, [vp, vp, vp, u64, i32, i32, i32, dbl, u64, u64, vp, u64, vp, u64, vp,
                                        C.POINTER(u64), C.POINTER(u64)]),
        "yttm_enc_run_subwords_device": (i32, [vp, vp, vp, u64, u64, i32, i32, i32, dbl, u64, u64, C.POINTER(vp),
                                               C.POINTER(vp), C.POINTER(vp), C.POINTER(u64), C.POINTER(u64)]),
        "yttm_enc_stream_begin": (i32, [vp, i32, i32, i32, dbl, u64, u64, i32, ENC_SINK, vp]),
        "yttm_enc_stream_feed": (i32, [vp, vp, u64]),
        "yttm_enc_stream_end": (i32, [vp, C.POINTER(u64), C.POINTER(u64), C.POINTER(u64)]),
        "yttm_dec_run": (i32, [vp, vp, vp, u64, vp, u64, vp, u64, vp, C.POINTER(u64)]),
        "yttm_dec_run_device": (i32, [vp, vp, u64, vp, u64, vp, u64, C.POINTER(vp), C.POINTER(vp), C.POINTER(u64)]),
        "yttm_dec_stream_begin": (i32, [vp, i32, vp, u64, ENC_SINK, vp]),
        "yttm_dec_stream_feed": (i32, [vp, vp, u64]),
        "yttm_dec_stream_feed_ids": (i32, [vp, vp, u64, vp, u64]),
        "yttm_dec_stream_end": (i32, [vp, C.POINTER(u64), C.POINTER(u64), C.POINTER(u64)]),
    }
    missing = []
    for name, (res, args) in sig.items():
        try:
            f = getattr(L, name)
        except AttributeError:   # an older build of the library: reported when (and only when) the symbol is used
            missing.append(name)
            continue
        f.restype = res
        f.argtypes = args
    L._yttm_missing = missing
    return L


EXPORTED_SYMBOLS_DEVICE_ABI = [
    "yttm_ctx_create", "yttm_ctx_destroy", "yttm_last_error", "yttm_device_count", "yttm_stage_ms",
    "yttm_launch_count", "yttm_train_load_corpus", "yttm_train_feed_begin", "yttm_train_feed", "yttm_train_feed_end",
    "yttm_train_feed_words", "yttm_train_fed_words",
    "yttm_train_char_hist", "yttm_train_get_char_hist",
    "yttm_train_char_hist_devptr", "yttm_train_char_hist_refresh", "yttm_train_set_alphabet", "yttm_train_build",
    "yttm_train_export_words", "yttm_train_import_words", "yttm_train_dist_init", "yttm_train_dist_connect",
    "yttm_train_dist_word_table", "yttm_train_dist_export_words", "yttm_train_dist_import_words", "yttm_train_run", "yttm_train_dump_pairs",
    "yttm_train_scan_once", "yttm_train_synth_words", "yttm_enc_create", "yttm_enc_destroy", "yttm_enc_run",
    "yttm_enc_run_device", "yttm_enc_run_spans", "yttm_enc_run_spans_device", "yttm_enc_run_subwords",
    "yttm_enc_run_subwords_device", "yttm_enc_run_padded", "yttm_enc_run_padded_device", "yttm_enc_run_windows_device",
    "yttm_enc_stream_begin",
    "yttm_enc_stream_feed", "yttm_enc_stream_end", "yttm_dec_run", "yttm_dec_run_device", "yttm_dec_stream_begin",
    "yttm_dec_stream_feed", "yttm_dec_stream_feed_ids", "yttm_dec_stream_end",
]


class TrainStats(C.Structure):
    _fields_ = [("n_bytes", C.c_uint64), ("n_words", C.c_uint64), ("n_unique", C.c_uint64), ("n_tokens", C.c_uint64),
                ("n_pairs", C.c_uint64), ("table_capacity", C.c_uint64)]
