"""TEST-ONLY numpy stand-ins for quokka_b200.ops.JoinTable.probe_ordered and JoinTable.place (csrc/join.cu).  install() adds
them to the JoinTable of tests/cpu_shim.py, so DataStream.join(maintain_sort_order=...) runs through the planner, the executors
and the gloo exchange without a GPU.  The GPU tests compare both kernels with these, bit for bit."""
from __future__ import annotations

import numpy as np
import torch

from oracle import relops as R
from quokka_b200 import _lib as L

HOW_NAME = {L.JOIN_INNER: "inner", L.JOIN_LEFT: "left", L.JOIN_SEMI: "semi", L.JOIN_ANTI: "anti"}


def ordered_pairs(probe_key: np.ndarray, build_key: np.ndarray, how: int):
    """(probe int32, build int32 | None) in the ordered probe's order: by probe row, a row's matches by build row."""
    li, ri = R.join_indices(probe_key.astype(np.int64), build_key.astype(np.int64), HOW_NAME[how])
    return li.astype(np.int32), (None if ri is None else ri.astype(np.int32))


def probe_ordered(table, key, how=L.JOIN_INNER, expect=None):
    """JoinTable.probe_ordered of the shim's JoinTable (its build keys in build-row order)."""
    bk = np.concatenate(table.keys) if table.keys else np.zeros(0, np.int64)
    li, ri = ordered_pairs(key.numpy(), bk, how)
    return torch.from_numpy(li), (None if ri is None else torch.from_numpy(ri))


def join_place(pos, nleft):
    """Received rows in left order: a stable sort by position (one position's rows are contiguous, so it keeps their order)."""
    p = pos.numpy()
    if len(p) and (p.min() < 0 or p.max() >= nleft):
        raise L.QkError("join_place: a position outside the left rows")
    src = np.argsort(p, kind="stable").astype(np.int32)
    return torch.from_numpy(src), torch.from_numpy(p[src].astype(np.int32))


def install():
    """Give the CPU stand-in's JoinTable the ordered probe and the placement.  Idempotent; it only adds methods, so programs
    that do not use them run as before, and on the GPU (where quokka_b200.ops is the real module) nothing reads them."""
    import cpu_shim
    cpu_shim.JoinTable.probe_ordered = probe_ordered
    cpu_shim.JoinTable.place = staticmethod(join_place)
