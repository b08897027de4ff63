"""Exact references and input generators for OrderedStream.shift (csrc/shift.cu, executors.ShiftExecutor).

The reference is pandas: `DataFrame.groupby(by, sort=False)[cols].shift(n)` over the rows in stream order, and a plain Python loop
when there is no key.  It knows nothing of partitions, inverse permutations or the numbering the kernel uses; tests translate."""
from __future__ import annotations

import numpy as np
import pandas as pd

HUGE = 1 << 40
SIZES = [0, 1, 2, 7, 1000, 65_537]


def reference_src(keys: np.ndarray | None, n: int, nrows: int) -> np.ndarray:
    """int64 per row: the row `n` places earlier (n > 0) / |n| later (n < 0) among the rows of its key, or -1."""
    if keys is None:
        out = np.full(nrows, -1, np.int64)
        for i in range(nrows):
            j = i - n
            if 0 <= j < nrows:
                out[i] = j
        return out
    if nrows == 0 or abs(n) >= nrows:
        return np.full(nrows, -1, np.int64) if n else np.arange(nrows, dtype=np.int64)
    df = pd.DataFrame({"k": keys, "r": np.arange(nrows, dtype=np.int64)})
    got = df.groupby("k", sort=False)["r"].shift(n)
    return got.fillna(-1).to_numpy().astype(np.int64)


def reference_shift(keys, n: int, values: dict, fill=None) -> dict:
    """{column: (values, validity uint8)} after the shift: pandas' groupby().shift(n, fill_value=...) where a fill is given."""
    nrows = len(next(iter(values.values()))[0]) if values else 0
    src = reference_src(keys, n, nrows)
    out = {}
    for c, (v, valid) in values.items():
        f = fill.get(c) if isinstance(fill, dict) else fill
        has = src >= 0
        o = np.where(has, v[np.maximum(src, 0)], v.dtype.type(0) if f is None else f).astype(v.dtype) if nrows else v.copy()
        ok = np.where(has, 1 if valid is None else valid[np.maximum(src, 0)], 0 if f is None else 1).astype(np.uint8) if nrows \
            else np.zeros(0, np.uint8)
        out[c] = (o, ok)
    return out


def pandas_shift(keys, n: int, v: np.ndarray, fill):
    """pandas' own answer for one column with a fill (the reference's form, used to check reference_shift itself)."""
    df = pd.DataFrame({"k": keys if keys is not None else np.zeros(len(v), np.int64), "v": v})
    return df.groupby("k", sort=False)["v"].shift(n, fill_value=fill).to_numpy()


def key_cases(nrows: int, seed: int = 0):
    """(name, int32 codes or None): one key, all-distinct keys, a few keys, 50 000 keys, and no key."""
    rng = np.random.default_rng(seed + nrows)
    return [("one-key", np.zeros(nrows, np.int32)), ("distinct", rng.permutation(nrows).astype(np.int32)),
            ("few", rng.integers(0, 7, nrows).astype(np.int32)), ("50k", rng.integers(0, 50_000, nrows).astype(np.int32)),
            ("none", None)]


def n_cases(nrows: int):
    return sorted({0, 1, -1, 3, -3, nrows, -nrows, HUGE, -HUGE})


def value_cases(nrows: int, seed: int = 1):
    """{dtype name: (values, validity or None)}: one column per kernel dtype, every second one with NULLs."""
    rng = np.random.default_rng(seed + nrows)
    mask = (rng.random(nrows) < 0.8).astype(np.uint8)
    return {"u8": (rng.integers(0, 256, nrows).astype(np.uint8), None),
            "i32": (rng.integers(-(1 << 31), 1 << 31, nrows).astype(np.int32), mask),
            "i64": (rng.integers(-(1 << 62), 1 << 62, nrows).astype(np.int64), None),
            "f32": (rng.standard_normal(nrows).astype(np.float32), mask), "f64": (rng.standard_normal(nrows), None)}


FILLS = {"u8": 7, "i32": -5, "i64": 1 << 40, "f32": 0.5, "f64": -2.25}
