"""The reference's Python surface (youtokentome/youtokentome.py:1-99 + the Cython class
youtokentome/cpp/yttm.pyx:52-181) over the CUDA library: same class, method names, argument
meaning, return types and exceptions (ValueError(status.message), TypeError for bad argument
types).  Additions are additive only: `encode_packed` (zero-marshalling numpy path, optionally with the source byte
span of every id), `encode_padded` (the same ids as padded, truncated [N, L] rows with their lengths),
`encode_windows` (the same ids as overlapping [W, L] windows of every sentence, with each row's sentence and start),
`encode_subwords_packed` (the subword pieces on the GPU), `encode_file` (a file of any size, line by line, to .npy files
or the CLI's id or subword text), `decode_packed` (the inverse of `encode_packed`, on the GPU), `decode_file` (the inverse of
`encode_file`: either of its outputs, of any size, back to text on the GPU), `count_words` / `train_from_counts` (a
corpus's word-count table, and training from such a table) and `dropout_seed`."""
import ctypes as C
import os
import sys
import threading
from collections import namedtuple
from collections.abc import Collection, Mapping, Sequence
from enum import Enum
from typing import List, Optional, Union

import numpy as np

from . import _lib


class OutputType(Enum):
    ID = 1
    SUBWORD = 2


def _pack(sentences):
    enc = [s.encode() if isinstance(s, str) else bytes(s) for s in sentences]
    offs = np.zeros(len(enc) + 1, dtype=np.uint64)
    if enc:
        np.cumsum([len(b) for b in enc], out=offs[1:])
    return b"".join(enc), offs


def _check_dropout(dropout_prob):  # yttm.pyx:92-93
    if dropout_prob < 0 or dropout_prob > 1:
        raise ValueError("dropout_prob value must be in the range [0, 1]. Current value of dropout_prob = " +
                         str(dropout_prob))


def _pad_arg(pad_id):
    """encode_padded / encode_windows' pad_id as the library takes it (None: the model's, YTTM_PAD_FROM_MODEL)."""
    if pad_id is None:
        return -2**63
    if isinstance(pad_id, bool) or not isinstance(pad_id, (int, np.integer)):
        raise TypeError("pad_id must be an int or None, not %s" % type(pad_id).__name__)
    pad = int(pad_id)
    if not -2**31 <= pad < 2**31:
        raise ValueError("pad_id must fit in int32. Current value of pad_id = %d" % pad)
    return pad


def _offsets_error(n_ids):  # the library's text for the same error
    return "decode: offsets must be non-decreasing and lie within the ids (n_ids = %d)" % n_ids


def _is_torch(x):
    return type(x).__module__.startswith("torch")


def _check_out(out):
    if out not in ("numpy", "torch", "cuda"):
        raise ValueError("out must be 'numpy', 'torch' or 'cuda'")


def _host_offsets(offsets):
    """offsets as contiguous numpy uint64, and n = len - 1."""
    if _is_torch(offsets):
        offsets = offsets.cpu().numpy()
    offsets = np.ascontiguousarray(offsets).astype(np.uint64, copy=False)
    if len(offsets) < 1:
        raise ValueError("offsets must hold at least one value")
    return offsets, len(offsets) - 1


def _stage_host(data, offsets):
    """A host batch as the library reads it: (keep-alive, byte pointer, byte count, uint64 offsets, n, pinned).  `data`:
    bytes-like, numpy array or CPU torch tensor."""
    pinned = False
    if _is_torch(data):
        data = data.contiguous()
        ptr, n_bytes, pinned = data.data_ptr(), data.numel(), data.is_pinned()
    elif isinstance(data, np.ndarray):
        data = np.ascontiguousarray(data)
        ptr, n_bytes = data.ctypes.data, data.nbytes
    else:
        data = data if isinstance(data, bytes) else bytes(data)
        ptr, n_bytes = C.cast(C.c_char_p(data), C.c_void_p), len(data)
    return (data, ptr, n_bytes) + _host_offsets(offsets) + (pinned,)


def _stage_device(data, offsets):
    """A batch on the current CUDA device, uploaded if needed: (device, data tensor, int64 offsets tensor, n)."""
    import torch
    dev = torch.device("cuda", torch.cuda.current_device())
    if _is_torch(data):
        d = data.to(dev, non_blocking=True).contiguous()
    elif isinstance(data, (bytes, bytearray, memoryview)):
        raw = bytearray(data)   # a writable copy: torch warns on read-only buffers
        d = (torch.frombuffer(raw, dtype=torch.uint8) if raw else torch.empty(0, dtype=torch.uint8)).to(dev)
    else:
        d = torch.from_numpy(np.require(data, requirements=["C", "W"])).to(dev)
    if _is_torch(offsets):
        d_offs = offsets.to(dev, dtype=torch.int64).contiguous()
    else:
        d_offs = torch.from_numpy(np.ascontiguousarray(offsets).astype(np.int64)).to(dev)
    if d_offs.numel() < 1:
        raise ValueError("offsets must hold at least one value")
    return dev, d, d_offs, d_offs.numel() - 1


def _stage_bytes(data, offsets):
    """_stage_device for encode: the library reads sentence 0 at the byte pointer it gets, so that pointer is the byte at
    offsets[0] and the byte count is offsets[n] - offsets[0].  Returns (device, keep-alive, pointer, byte count, int64
    offsets tensor, n)."""
    dev, d, d_offs, n = _stage_device(data, offsets)
    first, last = (int(v) for v in d_offs[[0, n]].cpu())
    return dev, d, d.data_ptr() + first, last - first, d_offs, n


def _outputs(res, out, unsigned):
    """Device results (CUDA tensors) as `out` asks: CUDA tensors, CPU tensors, or numpy arrays where the results at the
    indices `unsigned` (offsets and spans) become uint64."""
    if out == "cuda":
        return tuple(res)
    if out == "torch":
        return tuple(t.cpu() for t in res)
    return tuple(t.cpu().numpy().astype(np.uint64) if i in unsigned else t.cpu().numpy() for i, t in enumerate(res))


def _host_buffers(out, pinned, *specs):
    """Output buffers of a host call, one per (shape, numpy dtype): numpy arrays, or for out="torch" CPU tensors, pinned
    like the input, with uint64 as int64.  Returns (buffers, their pointers)."""
    if out == "torch":
        import torch
        dt = {np.int32: torch.int32, np.int64: torch.int64, np.uint64: torch.int64}
        bufs = [torch.empty(shape, dtype=dt[t], pin_memory=pinned) for shape, t in specs]
        return bufs, [b.data_ptr() for b in bufs]
    bufs = [np.empty(shape, dtype=t) for shape, t in specs]
    return bufs, [b.ctypes.data for b in bufs]


WordCounts = namedtuple("WordCounts", ["word_bytes", "word_offsets", "counts", "separators", "data_len"])
WordCounts.__doc__ = """A corpus's word-count table: word i is word_bytes[word_offsets[i]:word_offsets[i+1]] (uint8, uint64 offsets
from 0) occurring counts[i] times (uint64); `separators` separator units (space, \\t .. \\r, U+2581) and `data_len` decode
units in the text.  Training on it gives the model of training on the text."""


def _open_input(data, what):
    """(fd, fd to close or None, bytes or None) for a path, a file descriptor, an object with fileno() or bytes-like."""
    if isinstance(data, (str, os.PathLike)):
        try:
            fd = os.open(data, os.O_RDONLY | getattr(os, "O_CLOEXEC", 0))
        except OSError as e:
            raise ValueError("%s: cannot open '%s': %s" % (what, os.fsdecode(data), e.strerror)) from None
        return fd, fd, None
    if isinstance(data, int) and not isinstance(data, bool):
        return data, None, None
    if hasattr(data, "fileno"):
        return data.fileno(), None, None
    if isinstance(data, (bytes, bytearray, memoryview)):
        return -1, None, bytes(data)
    raise TypeError("data must be a path, a file descriptor, an object with fileno() or bytes-like, not %s" %
                    type(data).__name__)


def _int_array(x, name):
    """An integer numpy array or torch tensor -> (uint64 numpy array or int64 CUDA tensor, on_device); negative values
    raise ValueError."""
    if _is_torch(x):
        if x.dtype.is_floating_point or x.dtype.is_complex or x.dtype == __import__("torch").bool:
            raise TypeError("%s must hold integers, not %s" % (name, x.dtype))
        if x.numel() and bool((x < 0).any()):
            raise ValueError("%s must not be negative" % name)
        if x.is_cuda:
            import torch
            return x.to(torch.int64).contiguous(), True
        x = x.numpy()
    x = np.asarray(x)
    if x.dtype.kind not in "iu" and not (x.size == 0 and x.dtype.kind == "f"):
        raise TypeError("%s must hold integers, not %s" % (name, x.dtype))
    if x.dtype.kind == "i" and x.size and x.min() < 0:
        raise ValueError("%s must not be negative" % name)
    return np.ascontiguousarray(x.astype(np.uint64)).reshape(-1), False


def _pack_words(words):
    enc = []
    for w in words:
        if isinstance(w, str):
            enc.append(w.encode())
        elif isinstance(w, (bytes, bytearray, memoryview)):
            enc.append(bytes(w))
        else:
            raise TypeError("a word must be str or bytes, not %s" % type(w).__name__)
    offs = np.zeros(len(enc) + 1, dtype=np.uint64)
    if enc:
        np.cumsum([len(b) for b in enc], out=offs[1:])
    return np.frombuffer(b"".join(enc), dtype=np.uint8), offs


def _table_arrays(counts):
    """train_from_counts' `counts` other than a TSV path -> (bytes, offsets, counts, separators or None, on_device)."""
    if isinstance(counts, WordCounts):
        if counts.separators is not None and (not isinstance(counts.separators, (int, np.integer)) or
                                              isinstance(counts.separators, bool)):
            raise TypeError("separators must be an int or None, not %s" % type(counts.separators).__name__)
        b, offs, cnt = counts.word_bytes, counts.word_offsets, counts.counts
        seps = None if counts.separators is None else int(counts.separators)
        if all(_is_torch(t) and t.is_cuda for t in (b, offs, cnt)):
            import torch
            if b.dtype != torch.uint8:
                raise TypeError("word_bytes must be uint8, not %s" % b.dtype)
            offs, _ = _int_array(offs, "word_offsets")
            cnt, _ = _int_array(cnt, "counts")
            return b.contiguous(), offs, cnt, seps, True
        if _is_torch(b):
            b = b.cpu().numpy()
        b = np.ascontiguousarray(np.asarray(b))
        if b.dtype != np.uint8:
            raise TypeError("word_bytes must be uint8, not %s" % b.dtype)
        offs, _ = _int_array(offs.cpu() if _is_torch(offs) else offs, "word_offsets")
        cnt, _ = _int_array(cnt.cpu() if _is_torch(cnt) else cnt, "counts")
    elif isinstance(counts, Mapping):
        seps, words, vals = None, [], []
        for w, c in counts.items():
            if not isinstance(c, (int, np.integer)) or isinstance(c, bool):
                raise TypeError("a count must be an int, not %s" % type(c).__name__)
            if c < 0:
                raise ValueError("the count of %r is negative" % (w,))
            if w in ("", b""):
                seps = (seps or 0) + int(c)
                continue
            words.append(w)
            vals.append(int(c))
        if any(v >= 2 ** 64 for v in vals) or (seps or 0) >= 2 ** 64:
            raise ValueError("a count does not fit in 64 bits")
        b, offs = _pack_words(words)
        cnt = np.array(vals, dtype=np.uint64)
    elif isinstance(counts, (tuple, list)) and len(counts) == 2 and not isinstance(counts[0], (str, bytes)):
        words, c = counts
        if not isinstance(words, Sequence) or isinstance(words, (str, bytes)):
            raise TypeError("words must be a sequence of str or bytes, not %s" % type(words).__name__)
        if not (_is_torch(c) or isinstance(c, np.ndarray)):
            raise TypeError("counts must be a numpy array or a torch tensor, not %s" % type(c).__name__)
        b, offs = _pack_words(words)
        cnt, _ = _int_array(c.cpu() if _is_torch(c) else c, "counts")
        seps = None
    else:
        raise TypeError("counts must be a TSV path, a WordCounts, a dict or a pair (words, counts), not %s" %
                        type(counts).__name__)
    if len(offs) != len(cnt) + 1:
        raise ValueError("word_offsets must hold one value more than counts (%d and %d)" % (len(offs), len(cnt)))
    if len(offs) and int(offs[-1]) > len(b):
        raise ValueError("word_offsets pass the end of word_bytes")
    return b, offs, cnt, seps, False


class BPE:
    def __init__(self, model: str, n_threads: int = -1):
        self.model = model
        self.n_threads = n_threads
        self._open()

    def _open(self):
        L = _lib.lib()
        self._dev_lock = threading.Lock()   # device-resident results live in library memory until the next call
        self._h = L.yttm_api_open(self.model.encode(), self.n_threads)
        if not self._h:
            raise ValueError(L.yttm_api_last_error(None).decode())

    def __del__(self):
        h = getattr(self, "_h", None)
        if h:
            try:
                _lib.lib().yttm_api_close(h)
            except Exception:
                pass
            self._h = None

    def _err(self):
        return ValueError(_lib.lib().yttm_api_last_error(self._h).decode())

    @staticmethod
    def train(data: str, model: str, vocab_size: int, coverage: float = 1.0, n_threads: int = -1, pad_id: int = 0,
              unk_id: int = 1, bos_id: int = 2, eos_id: int = 3) -> "BPE":
        L = _lib.lib()
        rc = L.yttm_api_train(data.encode(), model.encode(), vocab_size, coverage, n_threads, pad_id, unk_id, bos_id,
                              eos_id)
        if rc != 0:
            raise ValueError(L.yttm_api_last_error(None).decode())
        return BPE(model=model, n_threads=n_threads)

    @staticmethod
    def count_words(data, output=None) -> WordCounts:
        """The word-count table of a corpus, counted on the GPU as BPE.train feeds it: `data` is a path, a file
        descriptor, an object with fileno() (a pipe works) or bytes-like.  Entries are sorted by count descending, then
        by bytes ascending.  With `output` (a path, "-" for stdout) the table is also written as TSV: the line
        "\\t<separators>", then one "word\\tcount" line per entry."""
        fd, opened, buf = _open_input(data, "count_words")
        sizes = np.zeros(4, dtype=np.uint64)
        L = _lib.lib()
        out = None if output is None else os.fsencode(output)
        try:
            if output is not None and os.fspath(output) == "-":
                sys.stdout.flush()
            rc = L.yttm_api_count_words(fd, buf, len(buf) if buf is not None else 0, out, sizes.ctypes.data)
        finally:
            if opened is not None:
                os.close(opened)
        if rc != 0:
            raise ValueError(L.yttm_api_last_error(None).decode())
        n, nb = int(sizes[0]), int(sizes[1])
        words = np.empty(nb, dtype=np.uint8)
        offs = np.empty(n + 1, dtype=np.uint64)
        cnt = np.empty(n, dtype=np.uint64)
        L.yttm_api_result_words(words.ctypes.data, offs.ctypes.data, cnt.ctypes.data)
        return WordCounts(words, offs, cnt, int(sizes[2]), int(sizes[3]))

    @staticmethod
    def train_from_counts(counts, model: str, vocab_size: int, coverage: float = 1.0, n_threads: int = -1,
                          pad_id: int = 0, unk_id: int = 1, bos_id: int = 2, eos_id: int = 3) -> "BPE":
        """Trains from a word-count table and writes the model BPE.train writes for any text with the same words,
        counts and separators (the same errors too).  `counts`: a TSV path as count_words writes it, a WordCounts
        (whose arrays may be CUDA tensors, read in place), a dict {word: count} whose key "" holds the separators, or a
        pair (words, counts) of str / bytes words and a numpy array or torch tensor.  Without separators there is one
        per occurrence."""
        L = _lib.lib()
        if isinstance(counts, (str, os.PathLike)):
            rc = L.yttm_api_train_counts(None, None, None, 0, 2 ** 64 - 1, 0, os.fsencode(counts), model.encode(),
                                         vocab_size, coverage, n_threads, pad_id, unk_id, bos_id, eos_id)
        else:
            b, offs, cnt, seps, on_device = _table_arrays(counts)
            if seps is not None and seps >= 2 ** 64 - 1:
                raise ValueError("separators must be below 2^64 - 1")
            ptr = (lambda t: t.data_ptr()) if on_device else (lambda a: a.ctypes.data)
            rc = L.yttm_api_train_counts(ptr(b), ptr(offs), ptr(cnt), len(cnt), 2 ** 64 - 1 if seps is None else seps,
                                         int(on_device), None, model.encode(), vocab_size, coverage, n_threads, pad_id,
                                         unk_id, bos_id, eos_id)
        if rc != 0:
            raise ValueError(L.yttm_api_last_error(None).decode())
        return BPE(model=model, n_threads=n_threads)

    def _run_device(self, dev, call, results):
        """Runs call() (a yttm_api_*_device call) and returns clones of what it published: results() lists (pointer,
        typestr, shape) once the call has set the counts.  The library's result buffers are reused by the next call on
        the handle, so they are copied under the lock."""
        import torch
        from .distributed import _DevView
        torch.cuda.synchronize()   # the library runs on its own stream
        with self._dev_lock:
            if call() != 0:
                raise self._err()
            res = []
            for ptr, ts, shape in results():
                k = int(np.prod(shape))
                res.append(torch.as_tensor(_DevView(ptr.value, k, ts), device=dev).view(shape).clone() if k else
                           torch.empty(shape, dtype={"|u1": torch.uint8, "<i4": torch.int32, "<i8": torch.int64}[ts],
                                       device=dev))
            torch.cuda.synchronize()
        return res

    # -- encode ---------------------------------------------------------------------------------
    def encode_packed(self, data, offsets, bos=False, eos=False, reverse=False, dropout_prob=0.0, out="numpy",
                      with_spans=False):
        """Additive fast path (no Python lists; replaces the marshalling of yttm.pyx:96-107): sentence i =
        data[offsets[i]:offsets[i+1]].  `data`: bytes / numpy uint8 / torch uint8 tensor (CPU or CUDA); `offsets`:
        uint64 array (or int64 tensor).  Returns (ids int32, id_offsets) as
          out="numpy"  numpy arrays (one call into buffers allocated here),
          out="torch"  CPU torch tensors (pinned if the input was),
          out="cuda"   CUDA torch tensors: input uploaded if needed, results stay on the device
                       (yttm_enc_run_device; nothing touches the host).
        with_spans=True returns (ids, id_offsets, spans) with the same ids: spans[j] = (start, end) of the bytes id j
        came from, in the coordinates of `offsets` (data[start:end]); shape (n_ids, 2), dtype and device of
        id_offsets.  An id covers a run of its word's units (code points or invalid bytes) and the invalid bytes
        between them; the word-initial "▁" and <BOS> / <EOS> have empty spans (yttm_enc_run_spans in yttm_b200.h)."""
        _check_out(out)
        _check_dropout(dropout_prob)
        L = _lib.lib()
        flags = (int(bos), int(eos), int(reverse), float(dropout_prob))
        if out == "cuda" or (_is_torch(data) and data.is_cuda):
            dev, keep, ptr, n_bytes, d_offs, n = _stage_bytes(data, offsets)
            p, total = [C.c_void_p() for _ in range(3)], C.c_uint64(0)
            args = (self._h, ptr, d_offs.data_ptr(), n_bytes, n) + flags + (C.byref(p[0]), C.byref(p[1]))
            if with_spans:
                res = self._run_device(dev, lambda: L.yttm_api_encode_spans_device(*args, C.byref(p[2]), C.byref(total)),
                                       lambda: [(p[0], "<i4", (total.value,)), (p[1], "<i8", (n + 1,)),
                                                (p[2], "<i8", (total.value, 2))])
            else:
                res = self._run_device(dev, lambda: L.yttm_api_encode_device(*args, C.byref(total)),
                                       lambda: [(p[0], "<i4", (total.value,)), (p[1], "<i8", (n + 1,))])
            return _outputs(res, out, (1, 2))
        keep, ptr, n_bytes, offsets, n, pinned = _stage_host(data, offsets)
        cap = int(n_bytes) + 3 * n + 16   # ids of a sentence of L bytes: at most L + 1 (+ <BOS> + <EOS>)
        specs = [((cap,), np.int32), ((n + 1,), np.uint64)] + ([((cap, 2), np.uint64)] if with_spans else [])
        bufs, ptrs = _host_buffers(out, pinned, *specs)
        total = C.c_uint64(0)
        args = (self._h, ptr, offsets.ctypes.data, n) + flags + (ptrs[0], cap, ptrs[1])
        if with_spans:
            rc = L.yttm_api_encode_spans_into(*args, ptrs[2], C.byref(total))
        else:
            rc = L.yttm_api_encode_ids_into(*args, C.byref(total))
        del keep
        if rc != 0:
            raise self._err()
        return (bufs[0][:total.value], bufs[1]) + ((bufs[2][:total.value],) if with_spans else ())

    def encode_padded(self, data, offsets, max_length=None, pad_id=None, bos=False, eos=False, reverse=False,
                      dropout_prob=0.0, out="numpy", with_spans=False):
        """encode_packed as model input, on the GPU: sentence i becomes row i of an [N, L] matrix.  With c_i = the ids
        encode_packed gives sentence i without bos / eos / reverse and K = L - bos - eos, row i is
        [<BOS>]? + c_i[:K] + [<EOS>]? (truncated at the end of the content, <BOS> / <EOS> kept), reversed as a whole
        with reverse, and its cells from len(row i) on hold the pad id.  L = max_length, or the longest row of the
        batch when max_length is None.  pad_id defaults to the model's <PAD> id.  Inputs as for encode_packed; dropout
        draws and the dropout_seed counter advance as in encode_packed.  Returns (ids int32 [N, L], lengths int64 [N])
        and with with_spans also spans [N, L, 2] (encode_packed's span of every kept id, [offsets[i+1], offsets[i+1])
        for pads) as numpy arrays (spans uint64), CPU torch tensors (out="torch") or CUDA tensors (out="cuda")."""
        _check_out(out)
        _check_dropout(dropout_prob)
        if max_length is not None:
            if isinstance(max_length, bool) or not isinstance(max_length, (int, np.integer)):
                raise TypeError("max_length must be an int or None, not %s" % type(max_length).__name__)
            max_length = int(max_length)
            if max_length < 1 or max_length < int(bos) + int(eos) or max_length >= 2**31:
                raise ValueError("max_length must be at least 1 and at least bos + eos, and below 2^31. Current value "
                                 "of max_length = %d" % max_length)
        pad = _pad_arg(pad_id)
        L = _lib.lib()
        flags = (int(bos), int(eos), int(reverse), float(dropout_prob))
        if out == "cuda" or (_is_torch(data) and data.is_cuda) or max_length is None:
            dev, keep, ptr, n_bytes, d_offs, n = _stage_bytes(data, offsets)
            p, w = [C.c_void_p() for _ in range(3)], C.c_uint32(0)
            res = self._run_device(
                dev, lambda: L.yttm_api_encode_padded_device(self._h, ptr, d_offs.data_ptr(), n_bytes, n, *flags,
                                                             max_length or 0, pad, int(with_spans), C.byref(p[0]),
                                                             C.byref(p[1]), C.byref(p[2]), C.byref(w)),
                lambda: [(p[0], "<i4", (n, w.value)), (p[1], "<i8", (n,))] +
                        ([(p[2], "<i8", (n, w.value, 2))] if with_spans else []))
            return _outputs(res, out, (2,))
        keep, ptr, _, offsets, n, pinned = _stage_host(data, offsets)
        W = max_length
        specs = [((n, W), np.int32), ((n,), np.int64)] + ([((n, W, 2), np.uint64)] if with_spans else [])
        bufs, ptrs = _host_buffers(out, pinned, *specs)
        rc = L.yttm_api_encode_padded_into(self._h, ptr, offsets.ctypes.data, n, *flags, W, pad, ptrs[0], ptrs[1],
                                           ptrs[2] if with_spans else None)
        del keep
        if rc != 0:
            raise self._err()
        return tuple(bufs)

    def encode_windows(self, data, offsets, max_length, stride=0, pad_id=None, bos=False, eos=False, reverse=False,
                       dropout_prob=0.0, out="numpy", with_spans=False):
        """encode_packed as overlapping windows of model input, on the GPU: instead of truncating a sentence, its ids
        are cut into windows of K = max_length - bos - eos content ids that overlap by `stride` ids (step
        D = K - stride).  With c_i = the ids encode_packed gives sentence i without bos / eos / reverse, sentence i gives
        one window if len(c_i) <= K, else 1 + ceil((len(c_i) - K) / D); window k holds c_i[k D : k D + K].  Every
        window becomes a row [<BOS>]? + content + [<EOS>]?, reversed as a whole with reverse, its cells from len(row)
        on holding the pad id (the model's <PAD> id unless pad_id is given); rows are in sentence order, then window
        order (yttm_enc_run_windows_device in yttm_b200.h gives the definition).  Inputs as for encode_packed, staged
        on the device; dropout draws once per word, as encode_packed does, and advances the dropout_seed counter the
        same way.  Returns (ids int32 [W, L], lengths int64 [W], sentence int64 [W], start int64 [W]): row r comes from
        sentence `sentence[r]` and its first content id is c_i[start[r]].  with_spans also returns spans [W, L, 2]
        (encode_packed's span of every content id, [offsets[i], offsets[i]) for <BOS>, [offsets[i+1], offsets[i+1])
        for <EOS> and pads), as numpy arrays (spans uint64), CPU torch tensors (out="torch") or CUDA tensors
        (out="cuda")."""
        _check_out(out)
        _check_dropout(dropout_prob)
        if isinstance(max_length, bool) or not isinstance(max_length, (int, np.integer)):
            raise TypeError("max_length must be an int, not %s" % type(max_length).__name__)
        max_length, be = int(max_length), int(bos) + int(eos)
        if max_length < be + 1 or max_length >= 2**31:
            raise ValueError("max_length must be at least bos + eos + 1, and below 2^31. Current value of max_length = "
                             "%d" % max_length)
        if isinstance(stride, bool) or not isinstance(stride, (int, np.integer)):
            raise TypeError("stride must be an int, not %s" % type(stride).__name__)
        stride = int(stride)
        if not 0 <= stride < max_length - be:
            raise ValueError("stride must be at least 0 and below max_length - bos - eos = %d. Current value of "
                             "stride = %d" % (max_length - be, stride))
        pad = _pad_arg(pad_id)
        L = _lib.lib()
        flags = (int(bos), int(eos), int(reverse), float(dropout_prob))
        p, rows = [C.c_void_p() for _ in range(5)], C.c_uint64(0)
        call = lambda ptr, d_offs, n_bytes, n: L.yttm_api_encode_windows_device(
            self._h, ptr, d_offs, n_bytes, n, *flags, max_length, stride, pad, int(with_spans),
            *[C.byref(x) for x in p], C.byref(rows))
        if not L.yttm_api_device_context(self._h):   # no CUDA device: the library says so, before anything is staged
            call(None, None, 0, 0)
            raise self._err()
        dev, keep, ptr, n_bytes, d_offs, n = _stage_bytes(data, offsets)
        res = self._run_device(
            dev, lambda: call(ptr, d_offs.data_ptr(), n_bytes, n),
            lambda: [(p[0], "<i4", (rows.value, max_length))] + [(p[i], "<i8", (rows.value,)) for i in (1, 2, 3)] +
                    ([(p[4], "<i8", (rows.value, max_length, 2))] if with_spans else []))
        return _outputs(res, out, (4,))

    def encode_subwords_packed(self, data, offsets, bos=False, eos=False, reverse=False, dropout_prob=0.0, out="numpy"):
        """encode(output_type=SUBWORD) of a packed batch on the GPU (inputs as for encode_packed).  Returns
        (piece_bytes uint8, piece_offsets, sentence_offsets): piece k = piece_bytes[piece_offsets[k]:piece_offsets[k+1]]
        as UTF-8, the pieces of sentence i = [sentence_offsets[i], sentence_offsets[i+1]); offsets are uint64 numpy
        arrays for out="numpy", int64 tensors for "torch" / "cuda"."""
        _check_out(out)
        _check_dropout(dropout_prob)
        L = _lib.lib()
        flags = (int(bos), int(eos), int(reverse), float(dropout_prob))
        if out == "cuda" or (_is_torch(data) and data.is_cuda):
            dev, keep, ptr, n_bytes, d_offs, n = _stage_bytes(data, offsets)
            p, n_p, n_b = [C.c_void_p() for _ in range(3)], C.c_uint64(0), C.c_uint64(0)
            res = self._run_device(
                dev, lambda: L.yttm_api_encode_subwords_device(self._h, ptr, d_offs.data_ptr(), n_bytes, n, *flags,
                                                               C.byref(p[0]), C.byref(p[1]), C.byref(p[2]),
                                                               C.byref(n_p), C.byref(n_b)),
                lambda: [(p[0], "|u1", (n_b.value,)), (p[1], "<i8", (n_p.value + 1,)), (p[2], "<i8", (n + 1,))])
            return _outputs(res, out, (1, 2))
        keep, ptr, n_bytes, offsets, n, _ = _stage_host(data, offsets)
        cap = int(n_bytes) + 3 * n + 16   # one piece per id
        # a piece is its units' bytes plus a leading U+2581 (3 bytes, at most one per word) or "<BOS>" / "<EOS>"
        bytes_cap = 4 * int(n_bytes) + 10 * n + 16
        text = np.empty(bytes_cap, dtype=np.uint8)
        po = np.empty(cap + 1, dtype=np.uint64)
        so = np.empty(n + 1, dtype=np.uint64)
        n_p, n_b = C.c_uint64(0), C.c_uint64(0)
        rc = L.yttm_api_encode_subwords_into(self._h, ptr, offsets.ctypes.data, n, *flags, text.ctypes.data, bytes_cap,
                                             po.ctypes.data, cap, so.ctypes.data, C.byref(n_p), C.byref(n_b))
        del keep
        if rc != 0:
            raise self._err()
        text, po = text[:n_b.value].copy(), po[:n_p.value + 1].copy()
        if out == "torch":
            import torch
            return torch.from_numpy(text), torch.from_numpy(po.astype(np.int64)), torch.from_numpy(so.astype(np.int64))
        return text, po, so

    def _pieces(self, need):
        """The calling thread's last length-framed piece list -> list of sentences, each a list of str."""
        L = _lib.lib()
        n_p, n_s = C.c_uint64(0), C.c_uint64(0)
        L.yttm_api_result_counts(self._h, C.byref(n_p), C.byref(n_s))
        buf = C.create_string_buffer(int(need) + 1)
        L.yttm_api_result_text(self._h, buf)
        po = np.zeros(n_p.value + 1, dtype=np.uint64)
        so = np.zeros(n_s.value + 1, dtype=np.uint64)
        L.yttm_api_result_offsets(self._h, po.ctypes.data, so.ctypes.data)
        raw, po, so = buf.raw, po.tolist(), so.tolist()
        pieces = [raw[po[i]:po[i + 1]].decode() for i in range(n_p.value)]
        return [pieces[so[i]:so[i + 1]] for i in range(n_s.value)]

    def encode(self, sentences: Union[str, List[str]], output_type: OutputType = OutputType.ID, bos: bool = False,
               eos: bool = False, reverse: bool = False, dropout_prob: float = 0):
        if not isinstance(output_type, OutputType):
            raise TypeError("parameter output_type must be youtokentome.OutputType, not %s}" % str(type(output_type)))
        _check_dropout(dropout_prob)
        single = isinstance(sentences, str)
        if not single:
            assert isinstance(sentences, (list, tuple))
        data, offs = _pack([sentences] if single else sentences)
        L = _lib.lib()
        if output_type == OutputType.ID:
            ids, oo = self.encode_packed(data, offs, bos, eos, reverse, dropout_prob)
            oo = oo.astype(np.int64)
            flat = ids.tolist()
            out = [flat[oo[i]:oo[i + 1]] for i in range(len(oo) - 1)]
        else:
            need = L.yttm_api_encode_subwords(self._h, data, offs.ctypes.data, len(offs) - 1, int(bos), int(eos),
                                              int(reverse), float(dropout_prob))
            if need < 0:
                raise self._err()
            out = self._pieces(need)
        return out[0] if single else out

    # -- tables ---------------------------------------------------------------------------------
    def vocab_size(self) -> int:
        return _lib.lib().yttm_api_vocab_size(self._h)

    def vocab(self) -> List[str]:
        return self._pieces(_lib.lib().yttm_api_vocab(self._h))[0]

    def subword_to_id(self, subword: str) -> int:
        return _lib.lib().yttm_api_subword_to_id(self._h, subword.encode())

    def id_to_subword(self, id: int) -> str:
        L = _lib.lib()
        need = L.yttm_api_id_to_subword(self._h, id)
        if need < 0:
            raise self._err()
        return self._pieces(need)[0][0]

    def decode(self, ids: Union[List[int], List[List[int]]], ignore_ids: Optional[Collection] = None) -> List[str]:
        if not isinstance(ids, list):  # yttm.pyx:138-146
            raise TypeError("{} is not a list instance".format(type(ids)))
        if not isinstance(ignore_ids, Collection) and ignore_ids is not None:
            raise TypeError("{} is not a Collection instance".format(type(ignore_ids)))
        if len(ids) > 0 and isinstance(ids[0], int):
            ids = [ids]
        ign = np.asarray(sorted(ignore_ids) if ignore_ids else [], dtype=np.int32)
        offs = np.zeros(len(ids) + 1, dtype=np.uint64)
        if ids:
            np.cumsum([len(s) for s in ids], out=offs[1:])
        flat = np.asarray([t for s in ids for t in s], dtype=np.int32)
        L = _lib.lib()
        need = L.yttm_api_decode(self._h, flat.ctypes.data, offs.ctypes.data, len(ids), ign.ctypes.data, len(ign))
        if need < 0:
            raise self._err()
        return [s[0] for s in self._pieces(need)]

    def decode_packed(self, ids, offsets, ignore_ids: Optional[Collection] = None, out="numpy"):
        """Additive GPU path of `decode` for a packed batch: sentence i = ids[offsets[i]:offsets[i+1]] (absolute
        indices, offsets[0] need not be 0).  `ids`: int32 / int64 numpy array or torch tensor (CPU or CUDA);
        `offsets`: uint64 / int64 array or tensor.  Returns (text_bytes uint8, text_offsets), text i =
        text_bytes[text_offsets[i]:text_offsets[i+1]] as UTF-8, the same text as decode(); as
          out="numpy"  numpy uint8 + uint64 arrays,
          out="torch"  CPU torch tensors (uint8 + int64),
          out="cuda"   CUDA torch tensors: ids uploaded if needed, results stay on the device."""
        _check_out(out)
        if not isinstance(ignore_ids, Collection) and ignore_ids is not None:
            raise TypeError("{} is not a Collection instance".format(type(ignore_ids)))
        ignore = sorted({int(i) for i in ignore_ids}) if ignore_ids else []
        L = _lib.lib()
        if out == "cuda" or (_is_torch(ids) and ids.is_cuda):
            import torch
            dev, d_ids, d_offs, n = _stage_device(ids, offsets)
            d_ids, extra = self._ids_int32(d_ids, lambda: d_offs.cpu().numpy().astype(np.uint64), ignore, torch)
            ign = np.asarray([i for i in ignore if -2**31 <= i < 2**31] + extra, dtype=np.int32)
            p_text, p_off, total = C.c_void_p(), C.c_void_p(), C.c_uint64(0)
            res = self._run_device(
                dev, lambda: L.yttm_api_decode_device(self._h, d_ids.data_ptr(), d_ids.numel(), d_offs.data_ptr(), n,
                                                      ign.ctypes.data, len(ign), C.byref(p_text), C.byref(p_off),
                                                      C.byref(total)),
                lambda: [(p_text, "|u1", (total.value,)), (p_off, "<i8", (n + 1,))])
            return _outputs(res, out, (1,))
        ids = ids.numpy() if _is_torch(ids) else np.asarray(ids)
        offsets, n = _host_offsets(offsets)
        if int(offsets[-1]) > len(ids):
            raise ValueError(_offsets_error(len(ids)))
        ids, extra = self._ids_int32(ids, lambda: offsets, ignore, np)
        ign = np.asarray([i for i in ignore if -2**31 <= i < 2**31] + extra, dtype=np.int32)
        total = C.c_uint64(0)
        cap = 8 * (int(offsets[-1]) - int(offsets[0])) + 64   # a first guess; the exact size on return code 2
        for _ in range(2):
            text = np.empty(max(cap, 1), dtype=np.uint8)
            oo = np.empty(n + 1, dtype=np.uint64)
            rc = L.yttm_api_decode_into(self._h, ids.ctypes.data, offsets.ctypes.data, n, ign.ctypes.data, len(ign),
                                        text.ctypes.data, cap, oo.ctypes.data, C.byref(total))
            if rc != 2:
                break
            cap = total.value
        if rc != 0:
            raise self._err()
        text = text[:total.value]
        if out == "torch":
            import torch
            return torch.from_numpy(text), torch.from_numpy(oo.astype(np.int64))
        return text, oo

    def _ids_int32(self, ids, offsets, ignore, xp):
        """ids as contiguous int32 (numpy, or torch on the ids' device) + values to add to the ignore list.  A value
        that does not fit in int32 is never truncated: if one is decoded (not ignored), the first invalid id of the
        batch raises decode's ValueError here; ignored ones become -1, which is then ignored as well.  `offsets()`
        gives the offsets as numpy uint64 (only needed on that rare path)."""
        if xp is np:
            if ids.dtype.kind not in "iu":
                raise TypeError("ids must be an integer array, not %s" % ids.dtype)
            if ids.dtype == np.int32:
                return np.ascontiguousarray(ids), []
            big = (ids < -2**31) | (ids > 2**31 - 1)
            if not big.any():
                return np.ascontiguousarray(ids.astype(np.int32)), []
            host = ids
        else:
            import torch
            if ids.dtype == torch.int32:
                return ids.contiguous(), []
            if ids.dtype.is_floating_point or ids.dtype.is_complex or ids.dtype == torch.bool:
                raise TypeError("ids must be an integer tensor, not %s" % ids.dtype)
            ids = ids.to(torch.int64)
            big = (ids < -2**31) | (ids > 2**31 - 1)
            if not bool(big.any()):
                return ids.to(torch.int32).contiguous(), []
            host = ids.cpu().numpy()
        offs = np.asarray(offsets(), dtype=np.uint64)
        lo, hi = int(offs[0]), int(offs[-1])
        if np.any(offs[1:] < offs[:-1]) or hi > len(host):
            raise ValueError(_offsets_error(len(host)))
        seen = np.asarray(host[lo:hi], dtype=np.int64)
        V = self.vocab_size()
        bad = np.flatnonzero(((seen < 0) | (seen >= V)) & ~np.isin(seen, np.asarray(ignore, dtype=np.int64)))
        if len(bad):
            raise ValueError("id must be in the range [0, vocab_size - 1]. Current value: vocab_size = %d; id=%d;"
                             % (V, int(seen[bad[0]])))
        if xp is np:
            return np.ascontiguousarray(np.where(big, -1, ids).astype(np.int32)), [-1]
        return torch.where(big, torch.full_like(ids, -1), ids).to(torch.int32).contiguous(), [-1]

    def encode_file(self, input, output, bos=False, eos=False, reverse=False, dropout_prob=0.0, text=False,
                    output_type: OutputType = OutputType.ID) -> dict:
        """Encodes a text file of any size on the GPU, line by line: a line ends at "\\n" and nowhere else, the text
        after the last "\\n" (if any) is a last line, and line i gets the ids encode_packed gives it without its
        "\\n".  Lines are the next sentences of the dropout stream, as for encode_packed.  `input`: a path, an int file
        descriptor or an object with fileno() (sys.stdin.buffer, a pipe), read to its end.  With output_type
        OutputType.ID, writes
          text=False  <output>.ids.npy (1-D uint16 when vocab_size() <= 65536, else int32) and <output>.offsets.npy
                      (uint64, lines + 1 values from 0: line i = ids[offsets[i]:offsets[i+1]]), both loadable with
                      np.load(..., mmap_mode="r");
          text=True   the text of `yttm encode --output_type id` (every id and one space, "\\n" per line) to
                      <output>, or to stdout when output is "-".
        OutputType.SUBWORD always writes text, whatever `text` says (it only chooses between the two id forms): the
        text of `yttm encode --output_type subword` (every piece encode_subwords_packed gives the line and one space,
        "\\n" per line) to <output>, or to stdout when output is "-".
        A failed call leaves nothing at the output names.  Returns {"lines", "ids", "bytes"} (bytes read; "ids" counts
        the pieces of the subword form, one per id)."""
        if not isinstance(output_type, OutputType):
            raise TypeError("parameter output_type must be youtokentome.OutputType, not %s}" % str(type(output_type)))
        _check_dropout(dropout_prob)
        subword = output_type == OutputType.SUBWORD
        output = os.fspath(output)
        opened = None
        if isinstance(input, (str, bytes, os.PathLike)):
            try:
                fd = opened = os.open(input, os.O_RDONLY | getattr(os, "O_CLOEXEC", 0))
            except OSError as e:
                raise ValueError("encode_file: cannot open '%s': %s" % (os.fsdecode(input), e.strerror)) from None
        elif isinstance(input, int) and not isinstance(input, bool):
            fd = input
        elif hasattr(input, "fileno"):
            fd = input.fileno()
        else:
            raise TypeError("input must be a path, a file descriptor or an object with fileno(), not %s" %
                            type(input).__name__)
        stats = np.zeros(3, dtype=np.uint64)
        try:
            if (text or subword) and output == "-":
                sys.stdout.flush()
            if subword:
                rc = _lib.lib().yttm_api_encode_file_subwords(self._h, fd, os.fsencode(output), int(bos), int(eos),
                                                              int(reverse), float(dropout_prob), stats.ctypes.data)
            else:
                rc = _lib.lib().yttm_api_encode_file(self._h, fd, os.fsencode(output), int(text), int(bos), int(eos),
                                                     int(reverse), float(dropout_prob), stats.ctypes.data)
        finally:
            if opened is not None:
                os.close(opened)
        if rc != 0:
            raise self._err()
        return {"lines": int(stats[0]), "ids": int(stats[1]), "bytes": int(stats[2])}

    def decode_file(self, input, output, ignore_ids: Optional[Collection] = None, text=False) -> dict:
        """Decodes ids of any size on the GPU, line by line, to what `yttm decode` prints for them: every line's decode
        followed by "\\n", to <output> or to stdout when output is "-".  `input`:
          text=False  the prefix of the pair encode_file writes (or np.save does): <input>.ids.npy, 1-D uint16 or int32,
                      and <input>.offsets.npy, 1-D uint64 from 0, non-decreasing, ending at len(ids): line i is
                      ids[offsets[i]:offsets[i+1]];
          text=True   id text (a path, an int file descriptor or an object with fileno(), read to its end), split into
                      lines as std::getline splits it; a line's ids are those `yttm decode` reads from it.
        ignore_ids as for decode.  A failed call leaves nothing at <output> (with "-", lines before the failing piece
        may have been written).  Returns {"lines", "ids", "bytes"} (text bytes written)."""
        if not isinstance(ignore_ids, Collection) and ignore_ids is not None:
            raise TypeError("{} is not a Collection instance".format(type(ignore_ids)))
        ign = np.asarray(sorted({int(i) for i in ignore_ids if -2**31 <= int(i) < 2**31}) if ignore_ids else [],
                         dtype=np.int32)
        output = os.fspath(output)
        opened, fd, prefix = None, -1, None
        if not text:
            if not isinstance(input, (str, bytes, os.PathLike)):
                raise TypeError("input must be the prefix of <input>.ids.npy and <input>.offsets.npy, not %s" %
                                type(input).__name__)
            prefix = os.fsencode(input)
        elif isinstance(input, (str, bytes, os.PathLike)):
            try:
                fd = opened = os.open(input, os.O_RDONLY | getattr(os, "O_CLOEXEC", 0))
            except OSError as e:
                raise ValueError("decode_file: cannot open '%s': %s" % (os.fsdecode(input), e.strerror)) from None
        elif isinstance(input, int) and not isinstance(input, bool):
            fd = input
        elif hasattr(input, "fileno"):
            fd = input.fileno()
        else:
            raise TypeError("input must be a path, a file descriptor or an object with fileno(), not %s" %
                            type(input).__name__)
        stats = np.zeros(3, dtype=np.uint64)
        try:
            if output == "-":
                sys.stdout.flush()
            rc = _lib.lib().yttm_api_decode_file(self._h, fd, prefix, os.fsencode(output), int(bool(text)),
                                                 ign.ctypes.data, len(ign), stats.ctypes.data)
        finally:
            if opened is not None:
                os.close(opened)
        if rc != 0:
            raise self._err()
        return {"lines": int(stats[0]), "ids": int(stats[1]), "bytes": int(stats[2])}

    # -- BPE-dropout stream ---------------------------------------------------------------------
    def dropout_seed(self, seed: int):
        """Reset the counter-based dropout generator (seed, sentence counter := 0)."""
        _lib.lib().yttm_api_set_dropout_seed(self._h, seed)

    # -- CLI helpers used by yttm_cli ------------------------------------------------------------
    def encode_cli(self, output_type, stream, bos, eos, reverse, dropout_prob):
        if _lib.lib().yttm_api_encode_cli(self._h, output_type.encode(), int(stream), int(bos), int(eos), int(reverse),
                                          float(dropout_prob)) != 0:
            raise self._err()

    def decode_cli(self, ignore_ids):
        ign = np.asarray(sorted(ignore_ids) if ignore_ids else [], dtype=np.int32)
        if _lib.lib().yttm_api_decode_cli(self._h, ign.ctypes.data, len(ign)) != 0:
            raise self._err()

    def vocab_cli(self, verbose):
        _lib.lib().yttm_api_vocab_cli(self._h, int(verbose))

    # -- pickling (youtokentome.py:90-99) ---------------------------------------------------------
    def __getstate__(self):
        return {"model": self.model, "n_threads": self.n_threads}

    def __setstate__(self, d):
        self.model = d["model"]
        self.n_threads = d["n_threads"]
        self._open()


def release_training_cache():
    """With YTTM_TRAIN_KEEP_CACHE=1 BPE.train keeps its device buffers (corpus, word table, packed words, pair table)
    cached per host thread so that repeated trainings do not reallocate; this gives the calling thread's back.  Without
    the variable every training frees them itself (the reference's train_bpe is stateless too)."""
    _lib.lib().yttm_api_release_training_cache()


def train_report():
    """Sizes / stage timings of the last BPE.train on this thread (dict)."""
    names = ["n_bytes", "data_len", "n_words", "n_unique", "n_tokens", "n_pairs", "n_merges", "read_s", "h2d_ms",
             "char_hist_ms", "word_count_ms", "tokenise_ms", "pair_hist_ms", "merge_loop_ms", "total_s", "launches",
             "loop_launches", "feed_pieces", "device_peak_bytes"]
    out = (C.c_double * len(names))()
    n = _lib.lib().yttm_api_train_report(out, len(names))
    return dict(zip(names[:n], list(out)[:n]))
