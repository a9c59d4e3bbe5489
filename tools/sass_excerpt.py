#!/usr/bin/env python
"""SASS evidence: opcode histogram + the hottest basic block (by static size heuristics: the longest run of
arithmetic between two branches) of one kernel in a built object.

    python tools/sass_excerpt.py urh_b200/build/digitize.o 'k_fsk_fifoILi4ELb0ELb1ELb1' > sass_k_fsk_fifo_stats.txt"""
import collections
import re
import subprocess
import sys


def main():
    obj, pat = sys.argv[1], sys.argv[2]
    txt = subprocess.run(["cuobjdump", "-sass", obj], stdout=subprocess.PIPE, text=True).stdout
    funcs = re.split(r"\n\s*Function : ", txt)
    body = None
    for f in funcs[1:]:
        name = f.split("\n", 1)[0].strip()
        if pat in name:
            body = f
            break
    if body is None:
        sys.exit("no function matching %r in %s" % (pat, obj))
    name = body.split("\n", 1)[0].strip()
    ins = []
    for line in body.split("\n"):
        m = re.match(r"\s*/\*([0-9a-f]{4,})\*/\s+(.*?);\s*/\*", line)
        if m:
            ins.append((m.group(1), m.group(2).strip()))
    ops = collections.Counter()
    for _, t in ins:
        t2 = re.sub(r"^@!?U?P\d+\s+", "", t)
        ops[t2.split()[0].split(".")[0]] += 1
    print("# %s\n# object %s, %d SASS instructions (static)" % (name, obj, len(ins)))
    print("# opcode histogram (static): " + ", ".join("%s %d" % kv for kv in ops.most_common(40)))
    marks = {"FMUL2": "packed f32x2 multiply", "FFMA2": "packed f32x2 fma", "FADD2": "packed f32x2 add", "UBLKCP": "TMA bulk copy",
             "SYNCS": "mbarrier", "LDG": "global load", "STG": "global store", "SHFL": "warp shuffle", "VOTE": "warp vote", "MUFU": "sfu"}
    print("# of note: " + ", ".join("%s=%d (%s)" % (k, ops[k], v) for k, v in marks.items() if ops.get(k)))
    # longest branch-free block
    best, cur, start = (0, 0), 0, 0
    for i, (_, t) in enumerate(ins):
        if re.search(r"\b(BRA|EXIT|RET|CALL|BSYNC|BSSY|WARPSYNC)\b", t):
            if i - start > best[0]:
                best = (i - start, start)
            start = i + 1
    n, st = best
    print("# longest branch-free block: %d instructions at /*%s*/ — first 120 shown" % (n, ins[st][0] if ins else "-"))
    for a, t in ins[st: st + min(n, 120)]:
        print("/*%s*/  %s" % (a, t))


if __name__ == "__main__":
    main()
