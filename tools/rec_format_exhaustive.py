#!/usr/bin/env python
"""Compare the float32 formatter (rechorus_b200/csrc/rec_format.cuh, through tests/rec_format_harness.cu) with NumPy's
repr on all 2^32 bit patterns, on every host core.  Takes about 15 minutes per style on 8 cores (NumPy's repr costs
about 1.5 us); prints one JSON summary line per style with the mismatch count and the first mismatches.

    python tools/rec_format_exhaustive.py [--styles 0,1] [--chunk-bits 22]
"""
import argparse
import json
import multiprocessing as mp
import os
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests import rec_csv_oracle as O  # noqa: E402

_exe = None
_work = None


def _init(exe, work):
    global _exe, _work
    _exe, _work = exe, tempfile.mkdtemp(dir=work)


def _chunk(args):
    lo, n, style = args
    bits = np.arange(lo, lo + n, dtype=np.uint64).astype(np.uint32)
    got = O.harness(_exe, bits, style, _work)
    want = O._repr_chunk((bits, style, False))
    bad = [(int(b), g, w) for b, g, w in zip(bits, got, want) if g != w]
    return len(bad), bad[:5]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--styles", default="0,1")
    ap.add_argument("--chunk-bits", type=int, default=22)
    a = ap.parse_args()
    with tempfile.TemporaryDirectory() as work:
        exe = O.build_harness(work)
        n = 1 << a.chunk_bits
        for style in (int(s) for s in a.styles.split(",")):
            t0 = time.time()
            with mp.get_context("fork").Pool(os.cpu_count() or 1, initializer=_init, initargs=(exe, work)) as pool:
                res = pool.map(_chunk, [(lo, n, style) for lo in range(0, 1 << 32, n)], chunksize=1)
            mismatches = sum(r[0] for r in res)
            first = [m for r in res for m in r[1]][:10]
            print(json.dumps({"style": "np" if style == O.STYLE_NP else "bare", "patterns": 1 << 32,
                              "mismatches": mismatches, "first": first, "seconds": round(time.time() - t0, 1),
                              "numpy": np.__version__}), flush=True)


if __name__ == "__main__":
    main()
