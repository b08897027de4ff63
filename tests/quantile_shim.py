"""TEST-ONLY numpy stand-in for quokka_b200.ops.QuantileSketch (csrc/quantile.cu), part of tests/cpu_shim.py, so that
DataStream.approximate_quantile runs through the planner, the executors and the gloo exchange without a GPU.  The sketch is
tests/quantile_cases.py's numpy restatement; the answers come from the product's own qsketch_quantiles (torch only)."""
from __future__ import annotations

import numpy as np
import torch

import quantile_cases as QC
from quokka_b200 import _lib as L
from quokka_b200 import ops as real_ops

_DTYPES = (torch.float64, torch.float32, torch.int64, torch.int32, torch.uint8)


class QuantileSketch:
    """The argument checks of qk_qsketch_update, the state as sorted numpy entries."""

    def __init__(self, k, device, capacity=1 << 16):
        self.k = int(k)
        if self.k < 1:
            raise L.QkError("QuantileSketch: k must be >= 1")
        e = np.zeros(0, dtype=np.uint64)
        self._e = (e, e.copy(), e.copy(), e.copy())
        self.rounds = self.grows = 0

    def _fold(self, key, cnt, mn, mx):
        key = np.concatenate([self._e[0], key])
        cnt = np.concatenate([self._e[1], cnt])
        mn = np.concatenate([self._e[2], mn])
        mx = np.concatenate([self._e[3], mx])
        uk, inv = np.unique(key, return_inverse=True)
        c = np.zeros(len(uk), dtype=np.uint64)
        np.add.at(c, inv, cnt)
        lo = np.full(len(uk), np.iinfo(np.uint64).max, dtype=np.uint64)
        np.minimum.at(lo, inv, mn)
        hi = np.zeros(len(uk), dtype=np.uint64)
        np.maximum.at(hi, inv, mx)
        self._e = (uk, c, lo, hi)

    def update(self, columns, valid=None):
        if len(columns) != self.k:
            raise L.QkError(f"QuantileSketch.update: {len(columns)} columns for a {self.k}-column sketch")
        if any(c.dtype not in _DTYPES for c in columns):
            raise L.QkError("qk_qsketch_update: bad dtype")
        n = columns[0].numel()
        if any(c.numel() != n for c in columns):
            raise L.QkError("qk_qsketch_update: columns of unequal length")
        masks = None if valid is None else [None if v is None else v.numpy() for v in valid]
        self._fold(*QC.sketch_entries([c.numpy() for c in columns], masks))

    def merge(self, keys, counts, mins, maxs):
        self._fold(*(t.numpy().view(np.uint64) for t in (keys, counts, mins, maxs)))

    def entries(self):
        return tuple(torch.from_numpy(a.view(np.int64).copy()) for a in self._e)

    def quantiles(self, qs):
        return real_ops.qsketch_quantiles(*self.entries(), self.k, qs)
