"""The reference's Python surface (youtokentome/youtokentome.py:1-99 + the Cython class
youtokentome/cpp/yttm.pyx:52-181) over the CUDA library: same class, method names, argument
meaning, return types and exceptions (ValueError(status.message), TypeError for bad argument
types).  Additions are additive only: `encode_packed` (zero-marshalling numpy path) and
`dropout_seed`."""
import ctypes as C
import threading
from collections.abc import Collection
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

    # -- encode ---------------------------------------------------------------------------------
    def encode_packed(self, data, offsets, bos=False, eos=False, reverse=False, dropout_prob=0.0, out="numpy"):
        """Additive fast path (no Python lists; replaces the marshalling of yttm.pyx:96-107): sentence i =
        data[offsets[i]:offsets[i+1]].  `data`: bytes / numpy uint8 / torch uint8 tensor (CPU or CUDA); `offsets`:
        uint64 array (or int64 tensor).  Returns (ids int32, id_offsets) as
          out="numpy"  numpy arrays (one call into buffers allocated here),
          out="torch"  CPU torch tensors (pinned if the input was),
          out="cuda"   CUDA torch tensors: input uploaded if needed, results stay on the device
                       (yttm_enc_run_device; nothing touches the host)."""
        L = _lib.lib()
        if out not in ("numpy", "torch", "cuda"):
            raise ValueError("out must be 'numpy', 'torch' or 'cuda'")
        is_torch = type(data).__module__.startswith("torch")
        if out == "cuda" or (is_torch and data.is_cuda):
            return self._encode_device(data, offsets, bos, eos, reverse, dropout_prob, out)
        keep = None
        if is_torch:
            keep = data = data.contiguous()
            ptr, n_bytes = data.data_ptr(), data.numel()
        elif isinstance(data, np.ndarray):
            keep = data = np.ascontiguousarray(data)
            ptr, n_bytes = data.ctypes.data, data.nbytes
        else:
            keep = data = bytes(data) if not isinstance(data, bytes) else data
            ptr, n_bytes = C.cast(C.c_char_p(data), C.c_void_p), len(data)
        if type(offsets).__module__.startswith("torch"):
            offsets = offsets.cpu().numpy()
        offsets = np.ascontiguousarray(offsets).astype(np.uint64, copy=False)
        n = len(offsets) - 1
        cap = int(n_bytes) + 3 * n + 16
        total = C.c_uint64(0)
        if out == "torch":
            import torch
            pin = is_torch and data.is_pinned()
            ids = torch.empty(cap, dtype=torch.int32, pin_memory=pin)
            oo = torch.empty(n + 1, dtype=torch.int64, pin_memory=pin)
            p_ids, p_oo = ids.data_ptr(), oo.data_ptr()
        else:
            ids = np.empty(cap, dtype=np.int32)
            oo = np.empty(n + 1, dtype=np.uint64)
            p_ids, p_oo = ids.ctypes.data, oo.ctypes.data
        rc = L.yttm_api_encode_ids_into(self._h, ptr, offsets.ctypes.data, n, int(bos), int(eos), int(reverse),
                                        float(dropout_prob), p_ids, cap, p_oo, C.byref(total))
        del keep
        if rc != 0:
            raise self._err()
        return ids[:total.value], oo

    def _encode_device(self, data, offsets, bos, eos, reverse, dropout_prob, out):
        import torch
        from .distributed import _DevView
        L = _lib.lib()
        dev = torch.device("cuda", torch.cuda.current_device())
        if type(data).__module__.startswith("torch"):
            d_bytes = data.to(dev, non_blocking=True).contiguous()
        else:
            raw = data if isinstance(data, (bytes, bytearray)) else np.ascontiguousarray(data).tobytes()
            d_bytes = torch.frombuffer(bytearray(raw), dtype=torch.uint8).to(dev)
        if type(offsets).__module__.startswith("torch"):
            d_offs = offsets.to(dev, dtype=torch.int64).contiguous()
        else:
            d_offs = torch.from_numpy(np.ascontiguousarray(offsets).astype(np.int64)).to(dev)
        n = d_offs.numel() - 1
        p_ids, p_off, total = C.c_void_p(), C.c_void_p(), C.c_uint64(0)
        torch.cuda.synchronize()   # the library runs on its own stream
        with self._dev_lock:       # the result pointers are valid until the next encode on this handle: copy under the lock
            rc = L.yttm_api_encode_device(self._h, d_bytes.data_ptr(), d_offs.data_ptr(), d_bytes.numel(), n, int(bos), int(eos),
                                          int(reverse), float(dropout_prob), C.byref(p_ids), C.byref(p_off), C.byref(total))
            if rc != 0:
                raise self._err()
            ids = torch.as_tensor(_DevView(p_ids.value, max(total.value, 1), "<i4"), device=dev)[:total.value].clone()
            oo = torch.as_tensor(_DevView(p_off.value, n + 1, "<i8"), device=dev).clone()
            torch.cuda.synchronize()
        if out == "cuda":
            return ids, oo
        if out == "torch":
            return ids.cpu(), oo.cpu()
        return ids.cpu().numpy(), oo.cpu().numpy().astype(np.uint64)

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
        if dropout_prob < 0 or dropout_prob > 1:  # yttm.pyx:92-93
            raise ValueError("dropout_prob value must be in the range [0, 1]. Current value of dropout_prob = " +
                             str(dropout_prob))
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
    out = (C.c_double * 16)()
    n = _lib.lib().yttm_api_train_report(out, 16)
    names = ["n_bytes", "data_len", "n_words", "n_unique", "n_tokens", "n_pairs", "n_merges", "read_s", "h2d_ms",
             "char_hist_ms", "word_count_ms", "tokenise_ms", "pair_hist_ms", "merge_loop_ms", "total_s", "launches"]
    return dict(zip(names[:n], list(out)[:n]))
