"""TEST-ONLY numpy stand-ins for quokka_b200.ops.shift_plan / shift_gather (csrc/shift.cu), part of tests/cpu_shim.py, so
OrderedStream.shift runs through the planner, the executors and the gloo exchange without a GPU.  The limits are the kernel's:
int32 row numbers, the five scalar dtypes."""
from __future__ import annotations

import numpy as np
import torch

from quokka_b200 import _lib as L

_DTYPES = (torch.uint8, torch.int32, torch.int64, torch.float32, torch.float64)
HUGE = 1 << 31


def shift_plan(n, nrows, by=None, n_by=0, dest=None, seg=None, lo=0, hi=None, want_edge=False, time=None, device=None):
    hi = nrows if hi is None else hi
    if nrows > 0x7fffffff:
        raise L.QkError("shift_plan: more than 2^31 - 1 rows")
    if (by is None) != (dest is None) or (by is None) != (seg is None):
        raise L.QkError("qk_shift_plan: by, dest and seg are given together or not at all")
    if not 0 <= lo <= hi <= nrows:
        raise L.QkError("qk_shift_plan: rows outside the input")
    sh = max(-HUGE, min(HUGE, int(n)))
    i = np.arange(nrows, dtype=np.int64)
    if by is None:
        p, s, e, inv = i, np.zeros(nrows, np.int64), np.full(nrows, nrows, np.int64), i
    else:
        p, sg, b = dest.numpy().astype(np.int64), seg.numpy(), by.numpy().astype(np.int64)
        s, e = sg[b], sg[b + 1]
        inv = np.empty(nrows, np.int64)
        inv[p] = i
    q = p - sh
    ok = (q >= s) & (q < e)
    row = np.where(ok, inv[np.clip(q, 0, max(nrows - 1, 0))] if nrows else q, -1)
    num = np.where(row >= lo, row - lo, row - lo + nrows)
    src = torch.from_numpy(np.where(ok, num, -1)[lo:hi].astype(np.int32))
    edge = None
    if want_edge:
        edge = torch.from_numpy((p >= e - sh if sh > 0 else (p < s - sh if sh < 0 else np.zeros(nrows, bool))).astype(np.uint8))
    bad = None
    if time is not None:
        t = time.numpy()
        has = p > s
        prev = inv[np.maximum(p - 1, 0)] if nrows else p
        bad = int((has & (t < t[prev])).sum()) if nrows else 0
    return src, edge, bad


def shift_gather(a, b, src, fills, a_valid=None, b_valid=None):
    nc, s = len(a), src.numpy().astype(np.int64)
    if nc == 0:
        return [], []
    a_valid = list(a_valid) if a_valid is not None else [None] * nc
    b_valid = list(b_valid) if b_valid is not None else [None] * nc
    outs, vouts = [], []
    for c in range(nc):
        if a[c].dim() != 1 or a[c].dtype not in _DTYPES:
            raise L.QkError(f"qk_shift_gather: unsupported column {a[c].dtype} with {a[c].dim()} dimensions")
        av = a[c].numpy()
        na = len(av)
        bv = b[c].numpy() if b is not None else np.zeros(0, av.dtype)
        if bv.dtype != av.dtype:
            raise L.QkError("qk_shift_gather: table B has another dtype")
        both = np.concatenate([av, bv])
        f = fills[c]
        o = np.where(s >= 0, both[np.maximum(s, 0)] if len(both) else np.zeros(len(s), av.dtype),
                     np.array(0 if f is None else f).astype(av.dtype)).astype(av.dtype)
        outs.append(torch.from_numpy(o))
        if f is None or a_valid[c] is not None or b_valid[c] is not None:
            va = a_valid[c].numpy() if a_valid[c] is not None else np.ones(na, np.uint8)
            vb = b_valid[c].numpy() if b_valid[c] is not None else np.ones(len(bv), np.uint8)
            vboth = (np.concatenate([va, vb]) != 0).astype(np.uint8)
            vouts.append(torch.from_numpy(np.where(s >= 0, vboth[np.maximum(s, 0)] if len(vboth) else 0,
                                                   0 if f is None else 1).astype(np.uint8)))
        else:
            vouts.append(None)
    return outs, vouts
