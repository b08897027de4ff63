"""TEST-ONLY numpy statements of quokka_b200.ops.JoinTable.probe_ordered and JoinTable.place (csrc/join.cu).  The JoinTable of
tests/cpu_shim.py answers with them, so DataStream.join(maintain_sort_order=...) runs through the planner, the executors and the
gloo exchange without a GPU.  The GPU tests compare both kernels with these, bit for bit."""
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


def join_place(pos, nleft):
    """Received rows in left order: a stable sort by position (one position's rows are contiguous, so it keeps their order)."""
    p = pos.numpy()
    if len(p) and (p.min() < 0 or p.max() >= nleft):
        raise L.QkError("join_place: a position outside the left rows")
    src = np.argsort(p, kind="stable").astype(np.int32)
    return torch.from_numpy(src), torch.from_numpy(p[src].astype(np.int32))

