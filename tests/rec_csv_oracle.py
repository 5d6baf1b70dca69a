"""What save_rec_results' CSV must contain, from NumPy and pandas themselves, and the sample of float32 bit patterns the
formatter (rechorus_b200/csrc/rec_format.cuh) is checked on.

  designed_sample()   >= 10^7 float32 bit patterns: every exponent's smallest, middle and largest mantissas, the
                      subnormals near 0 and below the normals, +-0, +-inf, NaNs with sign and payload bits, +-4096 ulps
                      around every power of ten from 1e-45 to 1e38, around both ends of the positional range of both
                      styles and around 2^24, then random patterns;
  numpy_repr(bits, style)   repr() of each np.float32 (or np.int64 with ints=True) in that style, on every core;
  build_harness(dir)  compiles tests/rec_format_harness.cu (host only) with nvcc and returns its path;
  harness(...)        runs it over an array and returns the lines;
  pandas_csv(...)     the bytes main.py:117-132's DataFrame.to_csv writes for (users, items, scores).
"""
from __future__ import annotations

import multiprocessing as mp
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
STYLE_NP, STYLE_BARE = 0, 1


def _f32_bits(x) -> int:
    return int(np.float32(x).view(np.uint32))


def designed_sample(n_total: int = 10_000_000, seed: int = 0) -> np.ndarray:
    """uint32 float bit patterns, the designed ones first, topped up with random patterns to n_total"""
    parts = []
    mant = np.array([0, 1, 2, 3, 0x400000 - 1, 0x400000, 0x400001, 0x7ffffd, 0x7ffffe, 0x7fffff], dtype=np.uint64)
    exps = np.arange(256, dtype=np.uint64)
    parts.append(((exps[:, None] << 23) | mant[None, :]).ravel())
    parts.append(np.arange(0, 1 << 18, dtype=np.uint64))                          # subnormals near 0 (and +0)
    parts.append(np.arange(0x7fffff - (1 << 16), 0x800000 + (1 << 16), dtype=np.uint64))   # largest subnormals
    parts.append(np.array([0x7f800000, 0x7f800001, 0x7fc00000, 0x7fc00001, 0x7fffffff, 0x7fa00000], dtype=np.uint64))
    centres = [_f32_bits(10.0 ** p) for p in range(-45, 39)]
    centres += [0x38d1b718, 0x49742400, 0x5a0e1bca, _f32_bits(2.0 ** 24)]          # 1e-4, 1e6, 1e16, 2^24
    w = np.arange(-4096, 4097, dtype=np.int64)
    for c in centres:
        v = np.int64(c) + w
        parts.append(v[(v >= 0) & (v < 0x7f800000)].astype(np.uint64))
    designed = np.concatenate(parts) & 0x7fffffff
    designed = np.concatenate([designed, designed | 0x80000000]).astype(np.uint32)   # both signs
    rest = max(0, n_total - designed.size)
    rnd = np.random.RandomState(seed).randint(0, 1 << 32, rest, dtype=np.uint64).astype(np.uint32)
    return np.concatenate([designed, rnd])


def int64_sample() -> np.ndarray:
    v = [0, 1, -1, np.iinfo(np.int64).max, np.iinfo(np.int64).min, np.iinfo(np.int64).max - 1,
         np.iinfo(np.int64).min + 1, 2 ** 32 - 1, 2 ** 32, 2 ** 32 + 1, -(2 ** 32), 2 ** 31, -(2 ** 31) - 1]
    for p in range(19):
        for d in (-1, 0, 1):
            v += [10 ** p + d, -(10 ** p + d)]
    rnd = np.random.RandomState(1).randint(np.iinfo(np.int64).min, np.iinfo(np.int64).max, 10000, dtype=np.int64)
    return np.concatenate([np.array(v, dtype=np.int64), rnd, rnd >> 33, rnd >> 50])


def _repr_chunk(args):
    values, style, ints = args
    arr = values.astype(np.int64) if ints else values.view(np.float32)
    if style == STYLE_BARE:
        with np.printoptions(legacy="1.25"):
            return [repr(x) for x in arr]
    return [repr(x) for x in arr]


def numpy_repr(values: np.ndarray, style: int, ints: bool = False) -> list:
    """repr() of np.float32(bits) (or np.int64 when ints) for every value, on every core"""
    chunks = np.array_split(values, max(1, min(64, values.size // 100_000)))
    if len(chunks) == 1:
        return _repr_chunk((values, style, ints))
    with mp.get_context("spawn").Pool(min(8, os.cpu_count() or 1)) as pool:        # no fork of a threaded process
        out = pool.map(_repr_chunk, [(c, style, ints) for c in chunks])
    return [s for part in out for s in part]


def build_harness(out_dir: str) -> str:
    exe = os.path.join(out_dir, "rec_format_harness")
    src = os.path.join(HERE, "rec_format_harness.cu")
    r = subprocess.run([NVCC, "-O2", "-std=c++17", "-x", "cu", src, "-o", exe], capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("nvcc failed on the harness:\n" + r.stdout + r.stderr)
    return exe


def harness(exe: str, values: np.ndarray, style: int, work_dir: str, ints: bool = False, raw: bool = False) -> list:
    """the harness's text for every value (uint32 float bits, or int64 when ints), as str lines (bytes when raw)"""
    src, dst = os.path.join(work_dir, "in.bin"), os.path.join(work_dir, "out.txt")
    np.ascontiguousarray(values, dtype=np.int64 if ints else np.uint32).tofile(src)
    subprocess.run([exe, "i64" if ints else "f32", str(style), src, dst], check=True)
    with open(dst, "rb") as f:
        text = f.read()
    lines = text.split(b"\n") if raw else text.decode("ascii").split("\n")
    assert not lines[-1]
    return lines[:-1]


def pandas_csv(path: str, users, items: np.ndarray, scores: np.ndarray, sep: str) -> bytes:
    """main.py:117-132's write of the lists (the DataFrame of Python lists of NumPy scalars)"""
    import pandas as pd
    rec_df = pd.DataFrame(columns=["user_id", "rec_items", "rec_predictions"])
    rec_df["user_id"] = users
    rec_df["rec_items"] = [list(r) for r in items]
    rec_df["rec_predictions"] = [list(r) for r in scores]
    rec_df.to_csv(path, sep=sep, index=False)
    with open(path, "rb") as f:
        return f.read()
