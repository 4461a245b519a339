"""ctypes bindings for the CHECKERS (test infrastructure): oracle/liboracle.so (our CPU
restatement) and oracle/_ref/libyttm_ref_{det,prod}.so (the unmodified reference compiled by
oracle/Makefile).  Only tests/, __graft_entry__.smoke() and bench.py's CPU legs import this."""
import atexit
import ctypes as C
import hashlib
import json
import lzma
import os
import subprocess
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_DIR = os.path.join(ROOT, "oracle")
ERRLEN = 1024


def build_checkers():
    """Compile oracle/liboracle.so and, when the reference sources exist (oracle/Makefile: REF), oracle/_ref/*.so."""
    subprocess.run(["make", "-s", "-C", ORACLE_DIR, "all"], check=True, stdout=subprocess.DEVNULL)


def _pack(sentences):
    """list[bytes] -> (concatenated bytes buffer, uint64 offsets[n+1])."""
    offs = np.zeros(len(sentences) + 1, dtype=np.uint64)
    if sentences:
        offs[1:] = np.cumsum([len(s) for s in sentences], dtype=np.uint64)
    return b"".join(sentences), offs


def _unpack(ids, offs):
    offs = offs.astype(np.int64)
    return [ids[offs[i]:offs[i + 1]].tolist() for i in range(len(offs) - 1)]


def read_model(path):
    """Model file (utils.cpp:50-91) -> (char2id dict, rules list[(x,y,z)], (unk,pad,bos,eos))."""
    with open(path) as f:
        tok = f.read().split()
    n, m = int(tok[0]), int(tok[1])
    p = 2
    c2i = {}
    for _ in range(n):
        c2i[int(tok[p])] = int(tok[p + 1])
        p += 2
    rules = []
    for _ in range(m):
        rules.append((int(tok[p]), int(tok[p + 1]), int(tok[p + 2])))
        p += 3
    special = tuple(int(x) for x in tok[p:p + 4])
    return c2i, rules, special


class _Enc:
    """Common encoder wrapper; subclasses set prefix / call conventions."""

    def __init__(self, lib, handle, prefix):
        self.lib, self.h, self.prefix = lib, handle, prefix

    def __del__(self):
        try:
            getattr(self.lib, self.prefix + "_encoder_free")(self.h)
        except Exception:
            pass

    def vocab_size(self):
        return getattr(self.lib, self.prefix + "_vocab_size")(self.h)


class Reference:
    """The unmodified reference (oracle/_ref).  kind: 'det' (parity) or 'prod' (timing)."""

    def __init__(self, kind="det"):
        path = os.path.join(ORACLE_DIR, "_ref", "libyttm_ref_%s.so" % kind)
        if not os.path.exists(path):
            raise FileNotFoundError(path)
        self.lib = lib = C.CDLL(path)
        lib.ref_train_file.argtypes = [C.c_char_p, C.c_char_p, C.c_int, C.c_double, C.c_int, C.c_int, C.c_int, C.c_int,
                                       C.c_int, C.POINTER(C.c_double), C.c_char_p, C.c_int]
        lib.ref_train_memory.argtypes = [C.c_char_p, C.c_uint64, C.c_char_p, C.c_int, C.c_double, C.c_int, C.c_int,
                                         C.c_int, C.c_int, C.c_int, C.POINTER(C.c_double), C.c_char_p, C.c_int]
        lib.ref_encoder_new.restype = C.c_void_p
        lib.ref_encoder_new.argtypes = [C.c_char_p, C.c_int, C.c_char_p, C.c_int]
        lib.ref_encoder_free.argtypes = [C.c_void_p]
        lib.ref_vocab_size.argtypes = [C.c_void_p]
        lib.ref_encode_ids.argtypes = [C.c_void_p, C.c_char_p, C.c_void_p, C.c_uint64, C.c_int, C.c_int, C.c_int,
                                       C.c_double, C.POINTER(C.c_double), C.POINTER(C.c_uint64), C.c_char_p, C.c_int]
        lib.ref_result_ids.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        lib.ref_encode_subwords.restype = C.c_int64
        lib.ref_encode_subwords.argtypes = [C.c_void_p, C.c_char_p, C.c_void_p, C.c_uint64, C.c_int, C.c_int, C.c_int,
                                            C.c_char_p, C.c_int64]
        lib.ref_decode_ids.restype = C.c_int64
        lib.ref_decode_ids.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_char_p, C.c_int64]
        self.deterministic = bool(lib.ref_is_deterministic_queue())

    def train(self, text, model_path, vocab_size, coverage=1.0, n_threads=1, pad=0, unk=1, bos=2, eos=3):
        """text: bytes.  Returns seconds; raises ValueError(Status.message)."""
        err = C.create_string_buffer(ERRLEN)
        sec = C.c_double(0)
        rc = self.lib.ref_train_memory(text, len(text), model_path.encode(), vocab_size, coverage, n_threads, pad, unk,
                                       bos, eos, C.byref(sec), err, ERRLEN)
        if rc != 0:
            raise ValueError(err.value.decode())
        return sec.value

    def train_file(self, input_path, model_path, vocab_size, coverage=1.0, n_threads=1, pad=0, unk=1, bos=2, eos=3):
        err = C.create_string_buffer(ERRLEN)
        sec = C.c_double(0)
        rc = self.lib.ref_train_file(input_path.encode(), model_path.encode(), vocab_size, coverage, n_threads, pad,
                                     unk, bos, eos, C.byref(sec), err, ERRLEN)
        if rc != 0:
            raise ValueError(err.value.decode())
        return sec.value

    def encoder(self, model_path, n_threads=1):
        err = C.create_string_buffer(ERRLEN)
        h = self.lib.ref_encoder_new(model_path.encode(), n_threads, err, ERRLEN)
        if not h:
            raise ValueError(err.value.decode())
        return RefEncoder(self.lib, h)


class RefEncoder(_Enc):
    def __init__(self, lib, h):
        super().__init__(lib, h, "ref")
        self.last_seconds = 0.0

    def encode_packed(self, buf, offs, bos=False, eos=False, reverse=False, dropout=0.0):
        err = C.create_string_buffer(ERRLEN)
        sec, tot = C.c_double(0), C.c_uint64(0)
        n = len(offs) - 1
        rc = self.lib.ref_encode_ids(self.h, buf, offs.ctypes.data, n, int(bos), int(eos), int(reverse), dropout,
                                     C.byref(sec), C.byref(tot), err, ERRLEN)
        if rc != 0:
            raise ValueError(err.value.decode())
        self.last_seconds = sec.value
        ids = np.zeros(max(tot.value, 1), dtype=np.int32)
        oo = np.zeros(n + 1, dtype=np.uint64)
        self.lib.ref_result_ids(self.h, ids.ctypes.data, oo.ctypes.data)
        return ids[:tot.value], oo

    def encode(self, sentences, **kw):
        buf, offs = _pack(sentences)
        ids, oo = self.encode_packed(buf, offs, **kw)
        return _unpack(ids, oo)

    def encode_subwords(self, sentences, bos=False, eos=False, reverse=False):
        buf, offs = _pack(sentences)
        need = self.lib.ref_encode_subwords(self.h, buf, offs.ctypes.data, len(sentences), int(bos), int(eos),
                                            int(reverse), None, 0)
        out = C.create_string_buffer(int(need) + 1)
        self.lib.ref_encode_subwords(self.h, buf, offs.ctypes.data, len(sentences), int(bos), int(eos), int(reverse),
                                     out, need)
        text = out.raw[:need].decode("utf-8", errors="replace")
        return [ln.split("\x01") if ln else [] for ln in text.split("\n")[:-1]]

    def decode(self, ids):
        a = np.asarray(ids, dtype=np.int32)
        need = self.lib.ref_decode_ids(self.h, a.ctypes.data, len(a), None, 0)
        out = C.create_string_buffer(int(need) + 1)
        self.lib.ref_decode_ids(self.h, a.ctypes.data, len(a), out, need)
        return out.raw[:need].decode("utf-8", errors="replace")


class Oracle:
    """oracle/liboracle.so — our CPU restatement."""

    def __init__(self):
        path = os.path.join(ORACLE_DIR, "liboracle.so")
        if not os.path.exists(path):
            build_checkers()
        self.lib = lib = C.CDLL(path)
        lib.orc_train_memory.argtypes = [C.c_char_p, C.c_uint64, C.c_char_p, C.c_int, C.c_double, C.c_int, C.c_int,
                                         C.c_int, C.c_int, C.POINTER(C.c_double), C.c_void_p, C.c_char_p, C.c_int]
        lib.orc_encoder_new.restype = C.c_void_p
        lib.orc_encoder_new.argtypes = [C.c_char_p, C.c_char_p, C.c_int]
        lib.orc_encoder_free.argtypes = [C.c_void_p]
        lib.orc_vocab_size.argtypes = [C.c_void_p]
        lib.orc_encode_ids.argtypes = [C.c_void_p, C.c_char_p, C.c_void_p, C.c_uint64, C.c_int, C.c_int, C.c_int,
                                       C.c_double, C.c_uint64, C.c_uint64, C.POINTER(C.c_double),
                                       C.POINTER(C.c_uint64), C.c_char_p, C.c_int]
        lib.orc_result_ids.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        lib.orc_train_words.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint32,
                                        C.c_uint32, C.c_void_p, C.c_void_p, C.POINTER(C.c_uint32)]
        lib.orc_words_state.argtypes = [C.c_void_p] * 5 + [C.POINTER(C.c_uint64)] * 3
        self.last_stats = None

    def train_words(self, tokens, offsets, freq, first_new_id, max_merges):
        """The merge loop on given words (word i = tokens[offsets[i]:offsets[i+1]], frequency freq[i]) ->
        list of (x, y, z, count at merge time)."""
        tokens = np.ascontiguousarray(tokens, dtype=np.uint32)
        offsets = np.ascontiguousarray(offsets, dtype=np.uint32)
        freq = np.ascontiguousarray(freq, dtype=np.uint64)
        rules = np.zeros(3 * max(max_merges, 1), dtype=np.uint32)
        cnts = np.zeros(max(max_merges, 1), dtype=np.uint64)
        nd = C.c_uint32(0)
        assert self.lib.orc_train_words(tokens.ctypes.data, len(tokens), offsets.ctypes.data, freq.ctypes.data,
                                        len(freq), first_new_id, max_merges, rules.ctypes.data, cnts.ctypes.data,
                                        C.byref(nd)) == 0, "orc_train_words: bad offsets"
        return [tuple(int(v) for v in rules[3 * i:3 * i + 3]) + (int(cnts[i]),) for i in range(nd.value)]

    def words_state(self):
        """After train_words: (tokens uint32, offsets uint64[n+1], freq uint64, keys uint64, counts uint64) — the words
        and the live pair table (key = x << 32 | y, count > 0)."""
        nw, nt, npr = C.c_uint64(0), C.c_uint64(0), C.c_uint64(0)
        self.lib.orc_words_state(None, None, None, None, None, C.byref(nw), C.byref(nt), C.byref(npr))
        tok = np.zeros(nt.value + 1, dtype=np.uint32)
        off = np.zeros(nw.value + 1, dtype=np.uint64)
        frq = np.zeros(nw.value + 1, dtype=np.uint64)
        keys = np.zeros(npr.value + 1, dtype=np.uint64)
        cnts = np.zeros(npr.value + 1, dtype=np.uint64)
        self.lib.orc_words_state(tok.ctypes.data, off.ctypes.data, frq.ctypes.data, keys.ctypes.data, cnts.ctypes.data,
                                 C.byref(nw), C.byref(nt), C.byref(npr))
        return tok[:nt.value], off, frq[:nw.value], keys[:npr.value], cnts[:npr.value]

    def train(self, text, model_path, vocab_size, coverage=1.0, pad=0, unk=1, bos=2, eos=3):
        err = C.create_string_buffer(ERRLEN)
        sec = C.c_double(0)
        stats = np.zeros(5, dtype=np.uint64)
        rc = self.lib.orc_train_memory(text, len(text), model_path.encode(), vocab_size, coverage, pad, unk, bos, eos,
                                       C.byref(sec), stats.ctypes.data, err, ERRLEN)
        if rc != 0:
            raise ValueError(err.value.decode())
        self.last_stats = dict(zip(["data_len", "n_words", "n_unique", "n_tokens", "n_merges"], stats.tolist()))
        return sec.value

    def encoder(self, model_path):
        err = C.create_string_buffer(ERRLEN)
        h = self.lib.orc_encoder_new(model_path.encode(), err, ERRLEN)
        if not h:
            raise ValueError(err.value.decode())
        return OracleEncoder(self.lib, h)


class OracleEncoder(_Enc):
    def __init__(self, lib, h):
        super().__init__(lib, h, "orc")
        self.last_seconds = 0.0

    def encode_packed(self, buf, offs, bos=False, eos=False, reverse=False, dropout=0.0, seed=0, first_index=0):
        err = C.create_string_buffer(ERRLEN)
        sec, tot = C.c_double(0), C.c_uint64(0)
        n = len(offs) - 1
        rc = self.lib.orc_encode_ids(self.h, buf, offs.ctypes.data, n, int(bos), int(eos), int(reverse), dropout, seed,
                                     first_index, C.byref(sec), C.byref(tot), err, ERRLEN)
        if rc != 0:
            raise ValueError(err.value.decode())
        self.last_seconds = sec.value
        ids = np.zeros(max(tot.value, 1), dtype=np.int32)
        oo = np.zeros(n + 1, dtype=np.uint64)
        self.lib.orc_result_ids(self.h, ids.ctypes.data, oo.ctypes.data)
        return ids[:tot.value], oo

    def encode(self, sentences, **kw):
        buf, offs = _pack(sentences)
        ids, oo = self.encode_packed(buf, offs, **kw)
        return _unpack(ids, oo)


class ReferenceReplay:
    """oracle/_ref/libyttm_ref_replay.so: the unmodified reference whose BPE-dropout draws are the product's Philox
    draws (oracle/replay_rng.h), one word at a time (oracle/ref_replay.cpp)."""

    def __init__(self, model_path=None):
        path = os.path.join(ORACLE_DIR, "_ref", "libyttm_ref_replay.so")
        if not os.path.exists(path):
            raise FileNotFoundError(path)
        self.lib = lib = C.CDLL(path)
        lib.rpl_open.restype = C.c_void_p
        lib.rpl_open.argtypes = [C.c_char_p, C.c_char_p, C.c_int]
        lib.rpl_close.argtypes = [C.c_void_p]
        lib.rpl_encode.argtypes = [C.c_void_p, C.c_char_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p,
                                   C.c_double, C.c_int, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64), C.c_char_p,
                                   C.c_int]
        lib.rpl_result.argtypes = [C.c_void_p] * 5
        lib.rpl_engine.argtypes = [C.c_uint64, C.c_uint64, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p]
        self.h = None
        if model_path is not None:
            err = C.create_string_buffer(ERRLEN)
            self.h = lib.rpl_open(model_path.encode(), err, ERRLEN)
            if not self.h:
                raise ValueError(err.value.decode())

    def __del__(self):
        if getattr(self, "h", None):
            self.lib.rpl_close(self.h)

    def encode_words(self, words, seeds, sents, word_offs, p, subwords=False):
        """Word i (bytes) under key (seeds[i], sents[i], word_offs[i]) -> {"ids": flat ids, "n": ids per word,
        "draws": draws per word, "pieces": per word the pieces joined by "\\x01" (with subwords)}."""
        buf, offs = _pack(words)
        seeds = np.ascontiguousarray(seeds, dtype=np.uint64)
        sents = np.ascontiguousarray(sents, dtype=np.uint64)
        word_offs = np.ascontiguousarray(word_offs, dtype=np.uint32)
        n_ids, n_text, err = C.c_uint64(0), C.c_uint64(0), C.create_string_buffer(ERRLEN)
        if self.lib.rpl_encode(self.h, buf, offs.ctypes.data, len(words), seeds.ctypes.data, sents.ctypes.data,
                               word_offs.ctypes.data, p, int(subwords), C.byref(n_ids), C.byref(n_text), err, ERRLEN):
            raise ValueError(err.value.decode())
        ids = np.zeros(n_ids.value + 1, dtype=np.int32)
        io = np.zeros(len(words) + 1, dtype=np.uint64)
        draws = np.zeros(len(words) + 1, dtype=np.uint32)
        text = C.create_string_buffer(n_text.value + 1)
        self.lib.rpl_result(self.h, ids.ctypes.data, io.ctypes.data, draws.ctypes.data, text)
        out = {"ids": ids[:n_ids.value].tolist(), "n": np.diff(io).tolist(), "draws": draws[:len(words)].tolist()}
        if subwords:
            out["pieces"] = text.raw[:n_text.value].decode("utf-8").split("\n")[:-1]
        return out

    def engine(self, seed, sent, word_off, n):
        """(2n raw engine words, n uniform_real_distribution<>(0, 1) draws) under one key."""
        words = np.zeros(2 * n, dtype=np.uint32)
        canon = np.zeros(n, dtype=np.float64)
        self.lib.rpl_engine(seed, sent, word_off, n, words.ctypes.data, canon.ctypes.data)
        return words.tolist(), canon.tolist()


def have_reference(kind="det"):
    return os.path.exists(os.path.join(ORACLE_DIR, "_ref", "libyttm_ref_%s.so" % kind))


# ---- stored answers of the reference ---------------------------------------------------------------------------
# The parity tests compare with the unmodified reference (DETERMINISTIC_QUEUE build).  Its answers to every call those
# tests make are stored in tests/golden/reference_answers.json.xz, keyed by a digest of the call's inputs, so that the
# comparison runs without the reference.  YTTM_REFERENCE_RECORD=<file> with oracle/_ref built runs the live reference
# and writes the stored answers plus its own to <file>.  Large id lists are stored as a digest and compare equal only to the same ids.
ANSWERS = os.path.join(ROOT, "tests", "golden", "reference_answers.json.xz")
_FULL_LIST_LIMIT = 4000   # characters of JSON; a longer list answer is stored as its digest


def _digest(*parts):
    h = hashlib.sha256()
    for p in parts:
        p = p if isinstance(p, bytes) else repr(p).encode()
        h.update(len(p).to_bytes(8, "little") + p)
    return h.hexdigest()[:32]


class ListDigest:
    """A stored list answer too long to keep: compares equal to the list it was taken from, and to nothing else."""

    def __init__(self, digest):
        self.digest = digest

    @staticmethod
    def of(value):
        return hashlib.sha256(json.dumps(value).encode()).hexdigest()[:32]

    def __eq__(self, other):
        return isinstance(other, list) and ListDigest.of(other) == self.digest

    def __repr__(self):
        return "ListDigest(%s)" % self.digest


class _Answers:
    def __init__(self):
        self.record = os.environ.get("YTTM_REFERENCE_RECORD")
        self.table, self.models = {}, {}
        if os.path.exists(ANSWERS):
            with lzma.open(ANSWERS, "rt") as f:
                d = json.load(f)
            self.table, self.models = d["calls"], d["models"]
        if self.record:
            atexit.register(self.save)

    def save(self):
        with lzma.open(self.record, "wb", preset=9 | lzma.PRESET_EXTREME) as f:
            f.write(json.dumps({"calls": self.table, "models": self.models}, sort_keys=True, separators=(",", ":")).encode())

    def get(self, key):
        if key not in self.table:
            raise LookupError("no stored reference answer for this call (record it with YTTM_REFERENCE_RECORD): " + key)
        return self.table[key]


_answers = None


def _store():
    global _answers
    if _answers is None:
        _answers = _Answers()
    return _answers


def _call(key, live, full=False):
    """The stored answer of `key`, or (recording) the live reference's, stored on the way: ("ok", value) / ("err", text).
    A long list is stored as {"digest": ...} and returned as a ListDigest, unless `full`."""
    st = _store()
    if st.record and have_reference("det"):
        try:
            value = live()
            if not full and isinstance(value, list) and len(json.dumps(value)) > _FULL_LIST_LIMIT:
                value = {"digest": ListDigest.of(value)}
            st.table[key] = ["ok", value]
        except ValueError as e:
            st.table[key] = ["err", str(e)]
    kind, value = st.get(key)
    if kind == "err":
        raise ValueError(value)
    return ListDigest(value["digest"]) if isinstance(value, dict) and "digest" in value else value


def _file_bytes(path):
    with open(path, "rb") as f:
        return f.read()


class StoredReference:
    """The reference's answers, from the live library while recording, else from tests/golden/reference_answers.json.xz."""

    def train(self, text, model_path, vocab_size, coverage=1.0, n_threads=1, pad=0, unk=1, bos=2, eos=3):
        args = (vocab_size, coverage, n_threads, pad, unk, bos, eos)
        return self._train("train", text, lambda: Reference("det").train(text, model_path, *args), model_path, args)

    def train_file(self, input_path, model_path, vocab_size, coverage=1.0, n_threads=1, pad=0, unk=1, bos=2, eos=3):
        args = (vocab_size, coverage, n_threads, pad, unk, bos, eos)
        return self._train("train_file", _file_bytes(input_path),
                           lambda: Reference("det").train_file(input_path, model_path, *args), model_path, args)

    @staticmethod
    def _train(kind, text, live_train, model_path, args):
        def live():
            live_train()
            model = _file_bytes(model_path)
            _store().models[_digest(model)] = model.decode("latin-1")   # a model file is ASCII text
            return {"model": _digest(model)}
        model = _store().models[_call(_digest(kind, text, *args), live)["model"]]
        with open(model_path, "wb") as f:
            f.write(model.encode("latin-1"))
        return 0.0

    def encoder(self, model_path, n_threads=1):
        return StoredRefEncoder(model_path, n_threads)

    def char2id_order(self, keys):
        """Slot order of the reference's char2id container after inserting `keys` in this order."""
        keys = np.ascontiguousarray(keys, dtype=np.uint32)

        def live():
            lib = Reference("det").lib
            lib.ref_char2id_order.restype = C.c_int
            lib.ref_char2id_order.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p]
            out = np.zeros(len(keys), dtype=np.uint32)
            assert lib.ref_char2id_order(keys.ctypes.data, len(keys), out.ctypes.data) == 0
            return out.tolist()
        return _call(_digest("char2id_order", keys.tobytes()), live)


class StoredRefEncoder:
    def __init__(self, model_path, n_threads):
        self.path, self.n_threads, self.model = model_path, n_threads, _file_bytes(model_path)
        _call(_digest("open", self.model), lambda: Reference("det").encoder(model_path, n_threads) and 0)

    def _live(self):
        return Reference("det").encoder(self.path, self.n_threads)

    def vocab_size(self):
        return _call(_digest("vocab_size", self.model), lambda: self._live().vocab_size())

    def encode(self, sentences, **kw):
        return _call(_digest("encode", self.model, *sentences, len(sentences), sorted(kw.items())),
                     lambda: self._live().encode(sentences, **kw))

    def encode_lengths(self, sentences, **kw):
        """Number of ids of every sentence (where a test needs no more of a long answer)."""
        return _call(_digest("encode_lengths", self.model, *sentences, len(sentences), sorted(kw.items())),
                     lambda: [len(s) for s in self._live().encode(sentences, **kw)], full=True)

    def encode_subwords(self, sentences, **kw):
        return _call(_digest("subwords", self.model, *sentences, len(sentences), sorted(kw.items())),
                     lambda: self._live().encode_subwords(sentences, **kw))

    def decode(self, ids):
        return _call(_digest("decode", self.model, np.asarray(ids, dtype=np.int64).tobytes()),
                     lambda: self._live().decode(ids))

    def replay_words(self, words, seeds, sents, word_offs, p, subwords=False):
        """ReferenceReplay.encode_words on this model (BPE-dropout with the product's draws)."""
        keys = np.stack([np.asarray(seeds, dtype=np.uint64), np.asarray(sents, dtype=np.uint64),
                         np.asarray(word_offs, dtype=np.uint64)]).tobytes() if len(words) else b""
        return _call(_digest("replay", self.model, *words, len(words), keys, float(p), bool(subwords)),
                     lambda: ReferenceReplay(self.path).encode_words(words, seeds, sents, word_offs, p, subwords))


def replay_engine(seed, sent, word_off, n):
    """ReferenceReplay.engine, stored like the reference's answers."""
    return _call(_digest("replay_engine", seed, sent, word_off, n),
                 lambda: list(ReferenceReplay().engine(seed, sent, word_off, n)), full=True)


def tmp_model_path(tag="m"):
    d = tempfile.mkdtemp(prefix="yttm_b200_")
    return os.path.join(d, tag + ".yttm")
