"""Fuzz the kernels under the SIMT emulator (tests/emul/simt; TEST HARNESS ONLY): random corpora x random
geometry (blocks, STREAMING window, ring depth, pair-table floor, deferred-list capacity, fed corpora in small pieces)
against the oracle.
usage: python tools/fuzz_emul.py [n_cases] [first_seed]"""
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402

import _bind  # noqa: E402
import _cases  # noqa: E402
from _bind import read_model, tmp_model_path  # noqa: E402
from _emu import emu_lib  # noqa: E402
from youtokentome_b200 import synth  # noqa: E402

KNOBS = ["YT_EMU_SMS", "YT_EMU_SCHED_SEED", "YTTM_FORCE_STREAM", "YTTM_STREAM_Q", "YTTM_STAGES", "YTTM_PAIR_CAP_FLOOR", "YTTM_DEFER_CAP",
         "YTTM_ENC_CHUNK_MB", "YTTM_ENC_DEDUP_SLOTS", "YTTM_ENC_DEDUP_WEAKTAG", "YTTM_XQ_SEG_CAP",
         "YTTM_PAIR_MAX_LOAD_PCT", "YTTM_FRONT_TOP", "YTTM_NEWP_LIMIT", "YTTM_DRAIN_PLACES", "YTTM_TRAIN_PIPELINE", "YTTM_TRAIN_PIPELINE_PIECE_KB", "YTTM_LOOP_THREADS",
         "YTTM_TRAIN_FEED_ABOVE", "YTTM_TRAIN_FEED_PIECE_KB"]


def sentences(rng, text):
    words = text.split() or [b"a"]
    out = []
    for _ in range(int(rng.integers(1, 120))):
        k = int(rng.integers(0, 40))
        s = b" ".join(words[int(i)] for i in rng.integers(0, len(words), k))
        r = int(rng.integers(0, 8))
        if r == 0:
            s = s + b" \xff\xfe\xe2\x96 "
        elif r == 1:
            s = b"  " + s.replace(b" ", b"\xe2\x96\x81", 2) + b"\t"
        elif r == 2:
            s = s + b" unseen-\xd1\x8f\xf0\x9f\x98\x80 zzz"
        elif r == 3 and words:
            s = b"".join(words[int(i)] for i in rng.integers(0, len(words), int(rng.integers(1, 400))))[:6000]  # one long word, often > 512
            # slots (capped: the ORACLE merges a word in O(n^2))
        out.append(s)
    return out + list(_cases.EDGE_SENTENCES)


def encode_case(rng, L, orc, model, text):
    import ctypes as C
    sents = sentences(rng, text)
    buf, offs = _bind._pack(sents)
    o = orc.encoder(model)
    h = L.yttm_api_open(model.encode(), 1)
    assert h
    try:
        for _ in range(3):
            kw = dict(bos=bool(rng.integers(0, 2)), eos=bool(rng.integers(0, 2)), reverse=bool(rng.integers(0, 2)))
            p = float(rng.choice([0.0, 0.0, 0.1, 0.5, 1.0]))
            seed = int(rng.integers(0, 2 ** 31))
            os.environ.pop("YTTM_ENC_DEDUP_WEAKTAG", None)
            if rng.integers(0, 2):
                os.environ["YTTM_ENC_DEDUP_WEAKTAG"] = "1"   # equal tags: every probe ends in the byte compare
            os.environ.pop("YTTM_ENC_DEDUP_SLOTS", None)
            if rng.integers(0, 2):
                os.environ["YTTM_ENC_DEDUP_SLOTS"] = str(int(rng.choice([1, 8, 64, 1024])))  # tiny tables: probe overflow
            want = o.encode(sents, dropout=p, seed=seed, **kw)
            L.yttm_api_set_dropout_seed(h, seed)
            total = C.c_uint64(0)
            rc = L.yttm_api_encode_ids(h, buf, offs.ctypes.data, len(sents), int(kw["bos"]), int(kw["eos"]),
                                       int(kw["reverse"]), p, C.byref(total))
            assert rc == 0, L.yttm_api_last_error(h)
            ids = np.zeros(max(total.value, 1), dtype=np.int32)
            oo = np.zeros(len(sents) + 1, dtype=np.uint64)
            L.yttm_api_result_ids(h, ids.ctypes.data, oo.ctypes.data)
            got = _bind._unpack(ids[:total.value], oo)
            if got != want:
                print("ENCODE MISMATCH", kw, p, seed, {k: os.environ.get(k) for k in KNOBS})
                return False
    finally:
        L.yttm_api_close(h)
    return True


def corpus(rng):
    kind = int(rng.integers(0, 7))
    if kind == 0:
        return synth.stress_text(int(rng.integers(0, 10 ** 6)))
    if kind == 1:
        return synth.readme_corpus(n_lines=int(rng.integers(5, 120)), n_chars=int(rng.integers(5, 120)),
                                   alphabet="abcd "[:int(rng.integers(2, 5))] + " ", seed=int(rng.integers(0, 999)))
    if kind == 2:
        return _cases.zipf().text(int(rng.integers(2000, 40000)), seed=int(rng.integers(0, 999)))
    if kind == 3:  # long runs and long words
        parts = [bytes([int(rng.choice(list(b"ab")))]) * int(rng.integers(1, 400)) for _ in range(int(rng.integers(2, 60)))]
        return b" ".join(parts) + b" " + b"ab" * int(rng.integers(1, 300))
    if kind == 4:
        return _cases.dirty_zipf_text(int(rng.integers(3000, 30000)))
    if kind == 5:  # every kind of separator, NUL, stray continuation / truncated bytes between short words
        alphabet = [b"a", b"b", b"ab", b"\x00", b"\t", b"\n", b"\r", b"\x0b", b"\x0c", b" ", b"\xe2\x96\x81", b"\xe2\x96", b"\x81",
                    b"\xff", b"\xc3\xa9", b"\xf0\x9f\x98\x80", b"\xf0\x9f", b"\xed\xa0\x80", b"\xc0\xaf", "я".encode(), "日".encode()]
        return b"".join(alphabet[int(i)] for i in rng.integers(0, len(alphabet), int(rng.integers(1, 3000))))
    # degenerate corpora
    return [b"", b" ", b"a", b"\xff", b"   \n\t ", b"aaaa", b"a a a a", b"\xe2\x96\x81", b"ab", "я".encode() * 3][int(rng.integers(0, 10))]


def main():
    n_cases = int(sys.argv[1]) if len(sys.argv) > 1 else 50
    first = int(sys.argv[2]) if len(sys.argv) > 2 else 0
    _bind.build_checkers()
    L, orc = emu_lib(), _bind.Oracle()
    t0 = time.time()
    for seed in range(first, first + n_cases):
        rng = np.random.default_rng(seed)
        text = corpus(rng)
        n_chars = len(set(text.decode("utf-8", "ignore")))
        vocab = n_chars + 4 + int(rng.integers(0, 120))
        cov = 1.0 if rng.integers(0, 2) else 1 - float(rng.random()) * 0.2
        env = {"YT_EMU_SMS": str(int(rng.integers(1, 5)))}
        if rng.integers(0, 2):
            env["YT_EMU_SCHED_SEED"] = str(int(rng.integers(1, 10 ** 6)))  # random fiber order inside every block
        if rng.integers(0, 3):
            env["YTTM_FORCE_STREAM"] = "1"
            env["YTTM_STREAM_Q"] = str(int(rng.choice([16, 32, 64, 100, 256, 1000, 4096])))
            env["YTTM_STAGES"] = str(int(rng.integers(2, 6)))
            if rng.integers(0, 2):
                env["YTTM_DEFER_CAP"] = str(int(rng.choice([1, 2, 5, 50])))
        if rng.integers(0, 2):
            env["YTTM_PAIR_CAP_FLOOR"] = str(int(rng.choice([16, 64, 256, 2048])))
        if rng.integers(0, 2):
            env["YTTM_XQ_SEG_CAP"] = str(int(rng.choice([4, 8, 64])))   # exchange segments overflow -> rebuild path
        if rng.integers(0, 3) == 0:
            env["YTTM_PAIR_MAX_LOAD_PCT"] = str(int(rng.choice([30, 50, 90])))
        # round 2: the replicated front (refresh rate, lost rounds), the drain geometry, the pipelined ingest
        if rng.integers(0, 2):
            env["YTTM_FRONT_TOP"] = str(int(rng.integers(1, 7)))
        if rng.integers(0, 2):
            env["YTTM_NEWP_LIMIT"] = str(int(rng.choice([1, 2, 5, 20, 768])))
        if rng.integers(0, 2):
            env["YTTM_DRAIN_PLACES"] = str(int(rng.integers(1, 8)))
        if rng.integers(0, 3) == 0:
            env["YTTM_TRAIN_PIPELINE"] = "1"
            env["YTTM_TRAIN_PIPELINE_PIECE_KB"] = str(int(rng.choice([1, 3, 16])))
        if rng.integers(0, 3) == 0:   # a fed corpus: pieces of 1 - 5 KB, merged into the persistent word table
            env["YTTM_TRAIN_FEED_ABOVE"] = str(int(rng.choice([0, 1000, 10000])))
            env["YTTM_TRAIN_FEED_PIECE_KB"] = str(int(rng.integers(1, 6)))
        if rng.integers(0, 3) == 0:
            env["YTTM_LOOP_THREADS"] = str(int(rng.choice([64, 128, 256])))
        for k in KNOBS:
            os.environ.pop(k, None)
        os.environ.update(env)
        m_o, m_e = tmp_model_path("fo"), tmp_model_path("fe")
        try:
            orc.train(text, m_o, vocab, cov)
            want = read_model(m_o)
        except ValueError as e:
            want = str(e)
        rc = L.yttm_api_train_memory(text, len(text), m_e.encode(), vocab, cov, 0, 1, 2, 3)
        got = read_model(m_e) if rc == 0 else L.yttm_api_last_error(None).decode()
        ok = got == want
        if ok and rc == 0:
            ok = encode_case(rng, L, orc, m_o, text)
        print("seed %d  %6d B  vocab %4d  cov %.3f  %s  %s" % (seed, len(text), vocab, cov, env, "ok" if ok else "MISMATCH"),
              flush=True)
        if not ok:
            sys.exit(1)
        for p in (m_o, m_e):
            if os.path.exists(p):
                os.remove(p)
    print("all %d cases ok in %.0f s" % (n_cases, time.time() - t0))


if __name__ == "__main__":
    main()
