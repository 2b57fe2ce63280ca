#!/usr/bin/env python
"""Medians of the `[kai]` profile lines of bench runs, per action kind, for before / after comparisons.

    KAI_PROFILE=1 python bench.py --gpus 1 --steps 25 --warmup 5 --parity off 2> before.err   # one build
    KAI_PROFILE=1 python bench.py --gpus 1 --steps 25 --warmup 5 --parity off 2> after.err    # the other
    python profiles/reclaim_ab.py before.err after.err

A solver action's lines start with its first `[kai] solver host profile` line, any other action's with its
`[kai] host-sequenced action` line; an action that printed the solver's set-up line is a solver action (reclaim at config3-cycle), the others are allocate.  Every number of every line is collected
in order, and the median over the actions of each kind is printed next to the line's text, so a field that a build
does not print shows as missing rather than as zero.  Warm-up steps are included: use enough steps to outvote them.
"""
import re
import statistics
import sys

NUM = re.compile(r"-?\d+(?:\.\d+)?")


def parse(path):
    kinds = {"allocate": [], "solver": []}
    cur = []

    def flush():
        if cur:
            solver = any(x.startswith("[kai] solver set-up") for x in cur)
            kinds["solver" if solver else "allocate"].append(list(cur))
            cur.clear()

    for line in open(path, errors="replace"):
        if not line.startswith("[kai]"):
            continue
        # a solver action starts with its first solver line; any action's block starts with its action line
        starts_solver = line.startswith("[kai] solver host profile:") and "simulations" in line
        starts_block = line.startswith("[kai] host-sequenced action")
        if starts_solver or (starts_block and any(x.startswith("[kai] host-sequenced action") for x in cur)):
            flush()
        cur.append(line.rstrip("\n"))
    flush()
    return kinds


def summary(actions):
    """{line template: [median of each number]} over the actions."""
    cols = {}
    for lines in actions:
        for line in lines:
            key = NUM.sub("#", line)
            cols.setdefault(key, []).append([float(x) for x in NUM.findall(line)])
    out = {}
    for key, rows in cols.items():
        width = min(len(r) for r in rows)
        out[key] = [statistics.median(r[i] for r in rows) for i in range(width)], len(rows)
    return out


def main(argv):
    runs = [(p, parse(p)) for p in argv[1:]]
    for kind in ("solver", "allocate"):
        print(f"== {kind} actions ==")
        for path, kinds in runs:
            acts = kinds[kind]
            print(f"-- {path}: {len(acts)} actions (medians)")
            for key, (med, n) in summary(acts).items():
                it = iter(f"{v:g}" for v in med)
                print("   " + NUM.sub(lambda m: next(it, m.group(0)), key.replace("#", "0")) + f"   [{n}]")


if __name__ == "__main__":
    main(sys.argv)
