"""TEST-ONLY numpy stand-in for quokka_b200.ops.GramState (csrc/gram.cu), part of tests/cpu_shim.py, so that DataStream.gramian /
covariance run through the planner, the executors and the gloo exchange without a GPU."""
from __future__ import annotations

import numpy as np
import torch

from quokka_b200 import _lib as L


class GramState:
    """The argument checks of qk_gram, fp64 products."""

    def __init__(self, k, device):
        self.k = int(k)
        if self.k < 1:
            raise L.QkError("GramState: k must be >= 1")
        self.gram = torch.zeros(self.k, self.k, dtype=torch.float64)
        self.sums = torch.zeros(self.k, dtype=torch.float64)
        self.n = 0

    def update(self, columns, shift=None, variant=0):
        if len(columns) != self.k:
            raise L.QkError(f"GramState.update: {len(columns)} columns for a {self.k}-column state")
        if any(c.dtype not in (torch.float64, torch.float32, torch.int32, torch.int64) for c in columns):
            raise L.QkError("qk_gram: unsupported dtype (f64, f32, i32 or i64)")
        n = columns[0].numel()
        if any(c.numel() != n for c in columns):
            raise L.QkError("qk_gram: columns of unequal length")
        x = np.stack([c.numpy().astype(np.float64) for c in columns], axis=1) if n else np.zeros((0, self.k))
        if shift is not None:
            x = x - shift.numpy()
        self.gram += torch.from_numpy(x.T @ x)
        self.sums += torch.from_numpy(x.sum(axis=0))
        self.n += n


def gram_last_plan():
    return "cpu-shim"
