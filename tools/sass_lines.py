"""Static instruction budget of one kernel: SASS instructions attributed to source lines (needs -lineinfo).

    cuobjdump -xelf all patchmatchnet_b200/libpmb200.so        (in a scratch directory)
    nvdisasm -g pm_kernels.sm_90a.cubin > pmk.sass
    python tools/sass_lines.py pmk.sass 'warp_corr3_kernelILi32ELi8ELi2ELi8ELi1ELi4E' [--ranges 700-733:phase1,...]

Counts are STATIC (one per SASS instruction, loops not weighted); inlined callee lines are reported with the innermost
file:line nvdisasm prints.  It is a budget for an issue-bound kernel, not a profile."""
import argparse
import collections
import re


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("sass")
    ap.add_argument("kernel")
    ap.add_argument("--ranges", default="")
    ap.add_argument("--top", type=int, default=40)
    args = ap.parse_args()
    text = open(args.sass).read().split("\n")
    start = None
    for i, l in enumerate(text):
        if l.startswith("\t.section\t.text.") and args.kernel in l:
            start = i
            break
    assert start is not None, "kernel not found"
    per_line = collections.Counter()
    per_op = collections.Counter()
    per_line_ops = collections.defaultdict(collections.Counter)
    cur = ("?", 0)
    n = 0
    for l in text[start + 1:]:
        if l.startswith("\t.section") or l.startswith("//-----"):
            break
        m = re.search(r'//## File "([^"]+)", line (\d+)', l)
        if m:
            # "inlined at" chains: keep the first (innermost) location printed for this instruction group
            cur = (m.group(1).split("/")[-1], int(m.group(2)))
            continue
        m = re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_.]+)", l)
        if m:
            op = m.group(1).split(".")[0]
            per_line[cur] += 1
            per_op[op] += 1
            per_line_ops[cur][op] += 1
            n += 1
    print(f"{n} SASS instructions")
    print("by opcode:", ", ".join(f"{k} {v}" for k, v in per_op.most_common(25)))
    if args.ranges:
        for spec in args.ranges.split(","):
            rng, name = spec.split(":")
            fname = None
            if "@" in rng:
                rng, fname = rng.split("@")
            lo, hi = map(int, rng.split("-"))
            tot = sum(v for (f, ln), v in per_line.items() if lo <= ln <= hi and (fname is None or f == fname))
            print(f"  {name:>28s} {spec.split(':')[0]:>24s}: {tot:5d}  ({100.0 * tot / n:4.1f} %)")
    print("top lines:")
    for (f, ln), v in per_line.most_common(args.top):
        ops = ", ".join(f"{k} {c}" for k, c in per_line_ops[(f, ln)].most_common(5))
        print(f"  {f}:{ln:<5d} {v:5d}   {ops}")


if __name__ == "__main__":
    main()
