"""A/B of the long-word encode path on one GPU (see DESIGN.md "Known weaknesses"):
    python tools/ab_long_words.py [word_bytes=16384] [n_words=8]
Encodes `n_words` sentences that are each ONE word of `word_bytes` random 'abcd' bytes with the default kernel
(one thread per word, O(n^2)) and with YTTM_ENC_LONG=1 (a block per word, a pass per rule); wall-clock ms of
yttm_api_encode_ids and a check that the ids are identical.  Keep word_bytes small at first: the default path is
quadratic (16 KB is expected to take about a second)."""
import ctypes as C
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402


def main(word_bytes=None, n_words=None):
    from youtokentome_b200 import synth
    from _gpu import GpuEncoder, gpu_train
    word_bytes = word_bytes or (int(sys.argv[1]) if len(sys.argv) > 1 else 16384)
    n_words = n_words or (int(sys.argv[2]) if len(sys.argv) > 2 else 8)
    model = gpu_train(synth.readme_corpus(n_lines=2000), 800, 1.0)
    rng = np.random.default_rng(1)
    sents = [bytes(rng.choice(list(b"abcd"), size=word_bytes).tolist()) for _ in range(n_words)]
    out, base = {}, None
    for name, env in (("default", None), ("YTTM_ENC_LONG", "1")):
        os.environ.pop("YTTM_ENC_LONG", None)
        if env:
            os.environ["YTTM_ENC_LONG"] = env
        g = GpuEncoder(model)
        g.encode(sents[:1])  # warm-up: allocations
        t0 = time.perf_counter()
        ids = g.encode(sents)
        ms = (time.perf_counter() - t0) * 1e3
        base = base or ids
        out[name] = {"ms": ms, "ids_equal_default": ids == base, "tokens_out": sum(len(x) for x in ids)}
    print(json.dumps({"word_bytes": word_bytes, "n_words": n_words, **out}, indent=1))
    return out


if __name__ == "__main__":
    main()
