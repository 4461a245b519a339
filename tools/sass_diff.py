"""Which kernels changed?  Compares two `cuobjdump -sass libyttm_b200.so` dumps function by function (whitespace
normalised: cuobjdump aligns columns to the longest line of the whole file).  Used to prove that adding an
experimental kernel or a test-only #ifdef leaves the measured kernels' machine code untouched.
    cuobjdump -sass youtokentome_b200/libyttm_b200.so > /tmp/new.sass ; python tools/sass_diff.py /tmp/old.sass /tmp/new.sass
Exits 0 only when both dumps hold the same functions with the same code.
--stats: for every changed function, the instruction counts and whether the opcode multisets are equal (a change
that only renumbers registers or reorders instructions keeps both)."""
import collections
import re
import sys


def functions(path):
    parts = re.split(r"\n\s*Function : ", open(path).read())
    out = {}
    for p in parts[1:]:
        name, body = p.split("\n", 1)
        # the anonymous-namespace hash (_cu_<hash>, or _GLOBAL__N__<hash>_ in CUDA 12.9) depends on the source text,
        # not only on its path; "identifier = <source path>" lines name the file, not code
        name = re.sub(r"_GLOBAL__N__[0-9a-f]{8}_", "_GLOBAL__N__", re.sub(r"_cu_[0-9a-f]{8}", "_cu_", name.strip()))
        out[name] = "\n".join(re.sub(r"\s+", " ", ln).strip() for ln in body.splitlines() if not ln.strip().startswith("identifier ="))
    return out


def opcodes(body):  # "/*0040*/ @!P0 IMAD.MOV.U32 R1, ..." -> "IMAD.MOV.U32"
    ops = (re.match(r"/\*[0-9a-f]{4,}\*/ (?:@!?U?P\w+ )?([A-Z][\w.]*)", ln) for ln in body.splitlines())
    return collections.Counter(m.group(1) for m in ops if m)


def main():
    args = [x for x in sys.argv[1:] if x != "--stats"]
    a, b = functions(args[0]), functions(args[1])
    for k in sorted(set(a) | set(b)):
        state = "only in new" if k not in a else "only in old" if k not in b else "same" if a[k] == b[k] else "CHANGED"
        print("%-12s %s" % (state, k[-90:]))
        if state == "CHANGED" and "--stats" in sys.argv:
            oa, ob = opcodes(a[k]), opcodes(b[k])
            print("             instructions %d -> %d, opcode multiset %s" %
                  (sum(oa.values()), sum(ob.values()), "equal" if oa == ob else "DIFFERS: %s" % ((oa - ob) + (ob - oa))))
    return 0 if a == b else 1


if __name__ == "__main__":
    sys.exit(main())
