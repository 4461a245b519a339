"""A plain restatement of encode_as_ids without dropout, from the parts of a model file: (char ids, rules, special
ids) as `_bind.read_model` returns them.  It shares no code with the kernels or with oracle/bpe_oracle.cpp, so the
tests can hand it models no trainer produces (a probe chain that wraps the rule table, duplicated pairs, U+2581 at
id 0 with long words) and still have an expectation.

The merge is the obvious one: the adjacent pair of minimum rule index, leftmost first, one merge at a time on a plain
list.  No passes and no rule about runs: "every second occurrence of x x x ..." must fall out of leftmost-first.
BPE-dropout is not restated; the dropout cases keep the oracle as their expectation."""
from _front_ref import SPACE_CP, byte_words, decode_units

_NONE = float("inf")
_UNK = -1   # a maximal run of out-of-alphabet characters: one token that no rule takes


def write_model(path, cp2id, rules, special):
    """The text format of a model file: counts, (code point, id) lines, (x, y, z) lines, unk pad bos eos."""
    with open(path, "w") as f:
        f.write("%d %d\n" % (len(cp2id), len(rules)))
        for cp, i in cp2id.items():
            f.write("%d %d\n" % (cp, i))
        for r in rules:
            f.write("%d %d %d\n" % tuple(r))
        f.write("%d %d %d %d\n" % tuple(special))
    return path


def rule_table(rules):
    """(x, y) -> (rule index, z) in file order: a later duplicate of a pair overwrites the earlier one."""
    rule2id = {}
    for k, (x, y, z) in enumerate(rules):
        rule2id[(x, y)] = (k, z)
    return rule2id


def encode_word(word, cp2id, rule2id, unk):
    """The ids of one byte-word (a maximal run of non-space bytes)."""
    t, last_unk = [cp2id[SPACE_CP]], False
    for _, _, cp in decode_units(word):
        if cp is None:
            continue                      # invalid units vanish
        if cp in cp2id:
            t.append(cp2id[cp])
            last_unk = False
        elif not last_unk:
            t.append(_UNK)
            last_unk = True
    if len(t) == 1:
        return []                         # no valid unit: no word
    rank = lambda i: rule2id.get((t[i], t[i + 1]), (_NONE, 0))[0]   # noqa: E731  ((_UNK, .) is in no rule)
    r = [rank(i) for i in range(len(t) - 1)]
    while r:
        best = min(r)
        if best == _NONE:
            break
        i = r.index(best)                 # leftmost
        t[i:i + 2] = [rule2id[(t[i], t[i + 1])][1]]
        del r[i]
        if i < len(r):
            r[i] = rank(i)
        if i > 0:
            r[i - 1] = rank(i - 1)
    if t[0] == 0 and cp2id[SPACE_CP] == 0:
        del t[0]                          # the id-0 quirk: a never-merged word-initial U+2581 whose id is 0 is left out
    return [unk if v == _UNK else v for v in t]


def encode(model, sentences, bos=False, eos=False, reverse=False, memo=None):
    """list[bytes] -> list[list[int]].  `memo` (a dict the caller keeps per model) remembers the ids of every distinct
    word, so that batches of many repeated words stay cheap."""
    cp2id, rules, (unk, _pad, bos_id, eos_id) = model
    memo = {} if memo is None else memo
    if "rule2id" not in memo:
        memo["rule2id"] = rule_table(rules)
    out = []
    for s in sentences:
        ids = [bos_id] if bos else []
        for w in byte_words(s):
            got = memo.get(w)
            if got is None:
                got = memo[w] = encode_word(w, cp2id, memo["rule2id"], unk)
            ids += got
        if eos:
            ids.append(eos_id)
        out.append(ids[::-1] if reverse else ids)
    return out
