"""BPE-dropout as the unmodified reference computes it, given the product's draws.

The product draws BPE-dropout decisions from Philox4x32-10: draw k of the word that starts at byte offset `off` of
sentence `sent` (counted from the handle's dropout_seed over every dropout call) is the first output word of
Philox4x32-10 with counter (sent lo, sent hi, off, k) and key (seed lo, seed hi), and the event it decides is skipped iff
that word / 2^32 < p.  oracle/_ref/libyttm_ref_replay.so runs the reference's own DropoutQueue on those draws, one word at
a time (oracle/ref_replay.cpp); `replayed` splits sentences into words with their keys and puts the words back
together with <BOS>, <EOS> and reverse, as encode_sentence does.  Its answers come through _bind.StoredReference, so
nothing here needs the reference at test time."""
from _bind import read_model
from _front_ref import SPACE_CPS, decode_units

M0, M1 = 0xD2511F53, 0xCD9E8D57
W0, W1 = 0x9E3779B9, 0xBB67AE85
MASK = 0xFFFFFFFF


def philox4x32_10(ctr, key):
    """Philox4x32-10 (Salmon et al., SC'11) of a counter of four and a key of two 32-bit words."""
    c0, c1, c2, c3 = ctr
    k0, k1 = key
    for _ in range(10):
        p0, p1 = M0 * c0, M1 * c2
        c0, c1, c2, c3 = ((p1 >> 32) ^ c1 ^ k0) & MASK, p1 & MASK, ((p0 >> 32) ^ c3 ^ k1) & MASK, p0 & MASK
        k0, k1 = (k0 + W0) & MASK, (k1 + W1) & MASK
    return c0, c1, c2, c3


def draw(seed, sent, word_off, k):
    """The word r of draw k of a word: the event is skipped iff r / 2^32 < p."""
    return philox4x32_10((sent & MASK, sent >> 32, word_off, k), (seed & MASK, seed >> 32))[0]


def sentence_words(sent):
    """[(byte offset, bytes)] of the words of one sentence: maximal runs of non-space units, invalid units included
    (they belong to the word they sit in, and a word may start with one), as the product keys its draws.  A word
    without a valid unit is kept too; the reference sees no word there and gives no ids."""
    out, start = [], None
    for p, n, cp in decode_units(sent) + [(len(sent), 0, 0x20)]:
        space = cp is not None and cp in SPACE_CPS
        if space and start is not None:
            out.append((start, sent[start:p]))
            start = None
        elif not space and start is None:
            start = p
    return out


def replay_batch(reference, model, sentences, p, seed, first_index, subwords=False):
    """The reference's ids (and pieces) of every word of the batch: (per sentence the list of word results)."""
    words, seeds, sents, offs, owner = [], [], [], [], []
    for i, s in enumerate(sentences):
        for off, w in sentence_words(s):
            words.append(w)
            seeds.append(seed)
            sents.append(first_index + i)
            offs.append(off)
            owner.append(i)
    r = reference.encoder(model).replay_words(words, seeds, sents, offs, p, subwords) if words else \
        dict(ids=[], n=[], draws=[], pieces=[])
    per = [[] for _ in sentences]
    pos = 0
    for j, i in enumerate(owner):
        ids = r["ids"][pos:pos + r["n"][j]]
        pos += r["n"][j]
        pieces = (r["pieces"][j].split("\x01") if r["pieces"][j] else []) if subwords else None
        per[i].append(dict(ids=ids, draws=r["draws"][j], pieces=pieces))
    return per


def replayed(reference, model, sentences, p, seed, first_index, bos=False, eos=False, reverse=False, subwords=False):
    """encode_as_ids (and with subwords encode_as_subwords) of the reference on `sentences`, the draws being those of
    sentence indices first_index, first_index + 1, ... under `seed`.  Returns ids per sentence, or (ids, pieces)."""
    _, _, (_, _, bos_id, eos_id) = read_model(model)
    ids, pieces = [], []
    for words in replay_batch(reference, model, sentences, p, seed, first_index, subwords):
        i = [bos_id] * bos + [x for w in words for x in w["ids"]] + [eos_id] * eos
        ids.append(i[::-1] if reverse else i)
        if subwords:
            q = ["<BOS>"] * bos + [x for w in words for x in w["pieces"]] + ["<EOS>"] * eos
            pieces.append(q[::-1] if reverse else q)
    return (ids, pieces) if subwords else ids

