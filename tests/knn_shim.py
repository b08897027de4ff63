"""TEST-ONLY numpy stand-ins for quokka_b200.ops.knn_topk / knn_merge (csrc/knn.cu), part of tests/cpu_shim.py, so that
DataStream.vector_nn_join runs through the planner, the executors and the gloo exchange without a GPU.  The gather and the
exchange of 2-D columns are cpu_shim's own (numpy fancy indexing moves whole rows)."""
from __future__ import annotations

import numpy as np
import torch

from quokka_b200 import _lib as L


def _better(sa, ka, sb, kb):
    return sa > sb or (sa == sb and ka < kb)


def knn_topk(x, probes, k):
    """The argument checks of qk_knn_topk; scores in fp64 rounded once to fp32, the kernel's selection rule."""
    if x.dim() != 2 or x.dtype not in (torch.float32, torch.float16):
        raise L.QkError("knn_topk: x must be an (n, d) f32 or f16 tensor")
    if probes.dim() != 2 or probes.dtype != torch.float32 or probes.shape[1] != x.shape[1]:
        raise L.QkError("knn_topk: probes must be a (q, d) fp32 tensor with the vectors' d")
    if not 1 <= k <= L.KNN_MAX_K:
        raise L.QkError(f"knn_topk: k must be in [1, {L.KNN_MAX_K}]")
    X = x.numpy().astype(np.float64)
    P = probes.numpy().astype(np.float64)
    with np.errstate(all="ignore"):
        n2 = (X * X).sum(axis=1)
        s = ((X @ P.T) / np.sqrt(n2)[:, None]).astype(np.float32)
    ok = np.isfinite(X).all(axis=1) & (n2 > 0)
    q = P.shape[0]
    scores = np.full((q, k), -np.inf, np.float32)
    rows = np.full((q, k), -1, np.int64)
    for p in range(q):
        idx = np.nonzero(ok & np.isfinite(s[:, p]))[0]
        order = idx[np.lexsort((idx, -s[idx, p].astype(np.float64)))][:k]
        scores[p, :len(order)] = s[order, p]
        rows[p, :len(order)] = order
    return torch.from_numpy(scores), torch.from_numpy(rows)


def knn_merge(a_score, a_key, b_score, b_key, k):
    q, ka, kb = a_score.shape[0], a_score.shape[1], b_score.shape[1]
    As, Ak, Bs, Bk = a_score.numpy(), a_key.numpy(), b_score.numpy(), b_key.numpy()
    os_ = np.full((q, k), -np.inf, np.float32)
    ok = np.full((q, k), -1, np.int64)
    src = np.full((q, k), -1, np.int32)
    for p in range(q):
        i = j = 0
        for o in range(k):
            ha, hb = i < ka and Ak[p, i] >= 0, j < kb and Bk[p, j] >= 0
            if not ha and not hb:
                break
            take_a = ha and not (hb and _better(Bs[p, j], Bk[p, j], As[p, i], Ak[p, i]))
            if take_a:
                os_[p, o], ok[p, o], src[p, o] = As[p, i], Ak[p, i], p * ka + i
                i += 1
            else:
                os_[p, o], ok[p, o], src[p, o] = Bs[p, j], Bk[p, j], q * ka + p * kb + j
                j += 1
    return torch.from_numpy(os_), torch.from_numpy(ok), torch.from_numpy(src)
