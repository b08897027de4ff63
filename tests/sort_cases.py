"""The exact reference and the case generators of the sort tests (numpy only; no GPU, no quokka_b200.ops).

The order is DuckDB's ORDER BY: integers by value, floats with -0.0 = +0.0 and every NaN after +inf, DESC the exact reverse of
that among non-NULL rows, NULL (valid == 0) after every valid row in BOTH directions and tied with each other; rows that tie
on every column keep their input order (stable).  `reference_perm_small` states those rules as a Python comparison, with no
use of the order image; `reference_perm` is np.lexsort over executors.order_image, for inputs too large for that, and the CPU
tests check the two against each other."""
from __future__ import annotations

import functools
import math

import numpy as np

TILE = 4096                       # csrc/sort.cu S_TILE: rows ranked in shared memory at a time
CHUNK_GRID = 264                  # chunks of a large input on a 132-SM H100 (two CTAs per SM)
DTYPES = (np.uint8, np.int32, np.int64, np.float32, np.float64)
SIZES = (0, 1, 2, 31, 32, 33, 255, 257, TILE - 1, TILE, TILE + 1, 2 * TILE, 3 * TILE + 5)
CHUNK_SIZES = (CHUNK_GRID * TILE - 1, CHUNK_GRID * TILE, CHUNK_GRID * TILE + 1)     # one tile per chunk / a second tile appears


def _cmp_values(a, b) -> int:
    """ascending comparison of two non-NULL values under the rules above"""
    fa, fb = isinstance(a, float), isinstance(b, float)
    na, nb = fa and math.isnan(a), fb and math.isnan(b)
    if na or nb:
        return int(na) - int(nb)
    return (a > b) - (a < b)              # -0.0 == 0.0 in Python as in SQL


def reference_perm_small(keys, valids, descending, dictionaries=None) -> np.ndarray:
    """Stable ORDER BY keys[0] [DESC], keys[1] [DESC], ... NULLS LAST -> row numbers in sorted order, by a Python comparison.
    A column with a dictionary is a string column of codes and sorts by the strings."""
    n = len(keys[0])
    cols = []
    for j, k in enumerate(keys):
        d = dictionaries[j] if dictionaries else None
        cols.append([d[int(c)] for c in k] if d is not None else [x.item() for x in k])

    def cmp(i, j):
        for c, v, desc in zip(cols, valids, descending):
            ni, nj = v is not None and v[i] == 0, v is not None and v[j] == 0
            if ni or nj:
                r = int(ni) - int(nj)
            else:
                r = _cmp_values(c[i], c[j])
                r = -r if desc else r
            if r:
                return r
        return 0
    return np.array(sorted(range(n), key=functools.cmp_to_key(cmp)), dtype=np.int32)


def reference_perm(keys, valids, descending, dictionaries=None) -> np.ndarray:
    """The same order by np.lexsort over the order images (for large inputs)."""
    from quokka_b200.executors import order_image
    lex = []
    for j, (k, v, desc) in enumerate(zip(keys, valids, descending)):
        d = dictionaries[j] if dictionaries else None
        if d is not None:
            k = np.argsort(np.argsort(np.array(d, dtype=object), kind="stable"), kind="stable")[k]
        img = order_image(np.asarray(k), desc)
        if v is not None:
            null = np.asarray(v) == 0
            img = np.where(null, np.uint64(0), img)
            lex.append(null)
        lex.append(img)
    return np.lexsort(lex[::-1]).astype(np.int32)


def sorted_image(key, valid, descending) -> np.ndarray:
    """What qk_sort_perm's image_out holds: the images in sorted order, a NULL row's being 0 (~0 when descending)."""
    from quokka_b200.executors import order_image
    img = order_image(np.asarray(key), descending)
    if valid is not None:
        img = np.where(np.asarray(valid) == 0, ~np.uint64(0) if descending else np.uint64(0), img)
    return img[reference_perm([key], [valid], [descending])]


def _floats(rng, n, dt):
    bits = {np.float32: (np.uint32, 0x7fc00001, 0xffc12345, 0x7f800001), np.float64: (np.uint64, 0x7ff8000000000001, 0xfff8123456789abc, 0x7ff0000000000001)}[dt]
    special = np.array([0.0, -0.0, np.inf, -np.inf, np.finfo(dt).tiny / 4, -np.finfo(dt).tiny / 4, np.finfo(dt).max, -np.finfo(dt).max, 1.5, -1.5], dtype=dt)
    nans = np.array(bits[1:], dtype=bits[0]).view(dt)                    # quiet and signalling NaNs of both signs with payloads
    pool = np.concatenate([special, nans, (rng.standard_normal(16) * 1e3).astype(dt)])
    return pool[rng.integers(0, len(pool), n)]


def key_cases(n: int, seed: int = 0):
    """(name, key) for every dtype and shape of data, n rows each."""
    rng = np.random.default_rng(seed + n)
    out = []
    for dt in DTYPES:
        name = np.dtype(dt).name
        if np.issubdtype(dt, np.floating):
            out.append((f"{name}-special", _floats(rng, n, dt)))
            out.append((f"{name}-random", (rng.standard_normal(n) * 1e6).astype(dt)))
        else:
            info = np.iinfo(dt)
            k = rng.integers(info.min, info.max, n, dtype=dt, endpoint=True)
            if n > 2:
                k[:2] = (info.min, info.max)
            out.append((f"{name}-full-range", k))
    i64 = np.int64
    out += [
        ("int32-dates", rng.integers(8035, 10561, n).astype(np.int32)),                         # ~2 500 distinct: two live digits
        ("int64-all-equal", np.full(n, 42, dtype=i64)),
        ("int64-sorted", np.arange(n, dtype=i64) - n // 2),
        ("int64-reversed", (np.arange(n, dtype=i64) * -3)),
        ("int64-two-values", rng.integers(0, 2, n).astype(i64) * 1000 - 7),
        ("int64-top-byte-only", rng.integers(-128, 128, n).astype(i64) << 56),
        ("int64-bottom-byte-only", rng.integers(0, 256, n).astype(i64) + (i64(0x1234) << 32)),
        ("float64-heavy-ties", rng.integers(0, 5, n).astype(np.float64) - 2.0),
    ]
    return out


def valid_cases(n: int, seed: int = 0):
    rng = np.random.default_rng(seed + 7 * n)
    return [("no-mask", None), ("some-null", (rng.random(n) < 0.7).astype(np.uint8)), ("all-null", np.zeros(n, np.uint8)),
            ("none-null", np.ones(n, np.uint8))]


def multi_column_case(n: int, ncols: int, seed: int = 0):
    """(keys, valids, descending, dictionaries): heavy ties in every column, mixed directions and dtypes, one string column
    whose dictionary order differs from its code order, NULLs in the second column."""
    rng = np.random.default_rng(seed + n + ncols)
    words = ["pear", "apple", "zebra", "Mango", "fig", "", "apple pie"]
    makers = [
        lambda: (rng.integers(0, 4, n).astype(np.int32), None, None),
        lambda: ((rng.integers(0, 3, n) - 1).astype(np.float64), (rng.random(n) < 0.8).astype(np.uint8), None),
        lambda: (rng.integers(0, len(words), n).astype(np.int32), None, words),
        lambda: (rng.integers(-2, 2, n).astype(np.int64), None, None),
    ]
    cols = [makers[j]() for j in range(ncols)]
    desc = [bool((seed + j) % 2) for j in range(ncols)]
    return [c[0] for c in cols], [c[1] for c in cols], desc, [c[2] for c in cols]


def assert_table_sorted_like(got: dict, table: dict, by, descending, valids=None, dictionaries=None, what=""):
    """`got` (column -> numpy array) must be `table` in reference order, row for row (a `rowid` column makes stability visible)."""
    keys = [table[c] for c in by]
    perm = reference_perm(keys, valids or [None] * len(by), descending, dictionaries)
    for c in table:
        a, b = np.asarray(got[c]), np.asarray(table[c])[perm]
        assert a.shape == b.shape, (what, c, a.shape, b.shape)
        same = (a == b) | ((a != a) & (b != b)) if a.dtype.kind == "f" else a == b
        assert bool(np.all(same)), f"{what}: column {c} differs at row {int(np.argmin(same))}"
