"""TEST-ONLY numpy stand-in for quokka_b200.ops.sort_perm (csrc/sort.cu), part of tests/cpu_shim.py, so that DataStream.sort
and what is built on it -- join_asof, windowed_transform, pattern_recognize over a sorted stream -- run through the planner,
the executors and the gloo exchange without a GPU.  The limits are the kernel's: the five scalar dtypes, int32 row numbers."""
from __future__ import annotations

import numpy as np
import torch

from quokka_b200 import _lib as L
from quokka_b200.executors import order_image

_DTYPES = (torch.uint8, torch.int32, torch.int64, torch.float32, torch.float64)
MAX_ROWS = 0x7fffffff


def sort_perm(key, valid, descending, perm_in=None, want_image=False):
    if key.dim() != 1 or key.dtype not in _DTYPES:
        raise L.QkError(f"qk_sort_perm: unsupported key {key.dtype} with {key.dim()} dimensions")
    n = key.numel()
    if n > MAX_ROWS:
        raise L.QkError("sort_perm: more than 2^31 - 1 rows")
    for t, dt in ((valid, torch.uint8), (perm_in, torch.int32)):
        if t is not None and (t.dtype != dt or t.numel() != n):
            raise L.QkError("sort_perm: masks and permutations have one entry per row")
    src = perm_in.numpy().astype(np.int64) if perm_in is not None else np.arange(n, dtype=np.int64)
    img = order_image(key.numpy()[src], bool(descending))
    null = np.zeros(n, bool) if valid is None else valid.numpy()[src] == 0
    img = np.where(null, ~np.uint64(0) if descending else np.uint64(0), img)
    order = np.lexsort((img, null))                                   # stable: ties keep the order of `src`
    perm = torch.from_numpy(src[order].astype(np.int32))
    return (perm, torch.from_numpy(img[order].view(np.int64).copy())) if want_image else perm


def sort_last_plan():
    return "cpu-shim"
