#!/usr/bin/env python
"""Compare two `bench.py --dump-outputs` directories array by array, bit for bit.

  python tools/compare_dumps.py DIR_A DIR_B

Both directories must hold the same arrays with the same shapes and dtypes, and every array must be bit-identical, with
one exception: a totalHits whose relation is GREATER_THAN_OR_EQUAL_TO is a lower bound that depends on the pruning order,
so `total_hits` is compared only where bit 0 of `flags` is clear in both dumps, and `conj_total_hits` only where
`conj_relation` is 0 in both. Exits 1 on any difference, 0 otherwise."""
import os
import sys

import numpy as np

# totals: the array that says where they are exact (EQUAL_TO), and how to read it
EXACT_WHERE = {"total_hits": ("flags", lambda f: (f.astype(np.int64) & 1) == 0),
               "conj_total_hits": ("conj_relation", lambda r: r == 0)}


def load(d):
    return {f[:-4]: np.load(os.path.join(d, f)) for f in sorted(os.listdir(d)) if f.endswith(".npy")}


def bits(a):
    return np.ascontiguousarray(a).view(np.uint8)


def main():
    if len(sys.argv) != 3:
        sys.exit(__doc__)
    a, b = load(sys.argv[1]), load(sys.argv[2])
    bad = [f"arrays differ: only in one dump: {sorted(set(a) ^ set(b))}"] if set(a) != set(b) else []
    for name in sorted(set(a) & set(b)):
        x, y = a[name], b[name]
        if x.shape != y.shape or x.dtype != y.dtype:
            bad.append(f"{name}: {x.dtype}{x.shape} vs {y.dtype}{y.shape}")
            continue
        if name in EXACT_WHERE and EXACT_WHERE[name][0] in a and EXACT_WHERE[name][0] in b:
            rel, exact = EXACT_WHERE[name]
            keep = exact(a[rel]) & exact(b[rel])
            x, y = x[keep], y[keep]
            what = f"{name} ({int(keep.sum())} of {keep.size} exact)"
        else:
            what = name
        diff = int((bits(x) != bits(y)).reshape(x.size, -1).any(axis=1).sum()) if x.size else 0
        print(f"{what}: {'identical' if diff == 0 else f'{diff} of {x.size} elements differ'}")
        if diff:
            bad.append(f"{name}: {diff} elements differ")
    for m in bad:
        print("DIFFERENT:", m, file=sys.stderr)
    sys.exit(1 if bad else 0)


if __name__ == "__main__":
    main()
