#!/usr/bin/env python
"""Nearest-neighbour benchmark (DataStream.vector_nn_join's kernel, qk_knn_topk in csrc/knn.cu) on one GPU; one JSON line on stdout.

  python tools/bench_knn.py [--rows 10000000] [--dim 768] [--probes 1,16,256,4096] [--k 10] [--reps 3] [--tiny]

Seeded vectors are generated on the device (N x d, f32 and f16; 10 M x 768 f32 is 30.7 GB).  For every probe count q the kernel
time comes from CUDA events over `reps` launches after a warm-up.  The roofline is the larger of the algorithmic bytes N d esize
over the HBM peak and the tensor-core flops over the dense TF32 peak, both H100 SXM data-sheet figures: 2 N d q per term, three
terms for f32 rows (3xTF32) and two for f16 rows (exact in TF32, two probe terms).  The same top-k from torch (chunked X @ P^T in fp32 with TF32 off, divided by the row norms, then
torch.topk) is timed alongside, and the two answers are compared outside the tie band of the error contract.  The card's name
and power limit are read in the same run.  Nothing is written to disk."""
from __future__ import annotations

import argparse
import json
import os
import sys

TOOLS = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(TOOLS))
sys.path.insert(0, TOOLS)                                                     # benchkit, also when loaded as a module

import torch

from benchkit import HBM_PEAK_TBS, card, event_ms
from quokka_b200 import ops

TF32_PEAK_TFLOPS = 495.0                       # H100 SXM data sheet (700 W card): TF32 tensor core, dense
TERMS = {"f32": 3, "f16": 2}                     # TF32 MMAs per product: 3xTF32 for f32 rows, two probe terms for f16 rows


def roofline(nbytes, flops, seconds):
    t_hbm, t_fp = nbytes / (HBM_PEAK_TBS * 1e12), flops / (TF32_PEAK_TFLOPS * 1e12)
    return {"bound": "hbm" if t_hbm >= t_fp else "tf32_tensor_core", "frac": max(t_hbm, t_fp) / seconds, "gb_per_s": nbytes / seconds / 1e9,
            "tflops": flops / seconds / 1e12, "algorithmic_bytes": nbytes, "algorithmic_flops": flops,
            "peaks": {"hbm_tb_per_s": HBM_PEAK_TBS, "tf32_tensor_core_tflops": TF32_PEAK_TFLOPS,
                      "source": "H100 SXM data sheet (700 W), not measured"}}


def torch_topk(x, phat, k, chunk_elems=1 << 29):
    """fp32 scores (TF32 off) chunk by chunk, torch.topk per chunk, then over the chunks' winners: (scores [q, k], rows [q, k])."""
    n, q = x.shape[0], phat.shape[0]
    step = max(1, chunk_elems // max(q, 1))
    best_s = torch.full((q, 0), float("-inf"), device=x.device)
    best_r = torch.zeros((q, 0), dtype=torch.int64, device=x.device)
    pt = phat.t().contiguous()
    for lo in range(0, n, step):
        xc = x[lo:lo + step].float()
        s = (xc @ pt) / xc.norm(dim=1, keepdim=True)
        s = torch.nan_to_num(s, nan=float("-inf"))
        v, i = torch.topk(s, min(k, s.shape[0]), dim=0)
        best_s = torch.cat([best_s, v.t()], dim=1)
        best_r = torch.cat([best_r, i.t() + lo], dim=1)
        v, j = torch.topk(best_s, min(k, best_s.shape[1]), dim=1)
        best_s, best_r = v, torch.gather(best_r, 1, j)
    return best_s, best_r


def agreement(x, phat, rows_a, rows_b, d):
    """Fraction of probes whose two top-k sets agree outside the tie band (rows in only one set score, in fp64, within
    2 (d + 8) 2^-21 of that probe's k-th fp64 score among the union)."""
    band = 2 * (d + 8) * 2.0 ** -21
    ok = 0
    q = phat.shape[0]
    for p in range(q):
        a = set(int(r) for r in rows_a[p].tolist() if r >= 0)
        b = set(int(r) for r in rows_b[p].tolist() if r >= 0)
        if a == b:
            ok += 1
            continue
        union = sorted(a | b)
        xs = x[union].double()
        s = ((xs @ phat[p].double()) / xs.norm(dim=1)).tolist()
        sc = dict(zip(union, s))
        kth = sorted(sc.values(), reverse=True)[min(len(a), len(b)) - 1]
        ok += all(abs(sc[r] - kth) <= band for r in a ^ b)
    return ok / q


def main(argv=None, dev=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--dim", type=int, default=768)
    ap.add_argument("--probes", default="1,16,256,4096")
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--dtypes", default="f32,f16")
    ap.add_argument("--tiny", action="store_true", help="4 096 x 64 vectors, q in {1, 17}: a quick check of the flow")
    a = ap.parse_args(argv)
    if a.tiny:
        a.rows, a.dim, a.probes = 4096, 64, "1,17"
    dev = dev or torch.device("cuda")
    torch.backends.cuda.matmul.allow_tf32 = False
    g = torch.Generator(device=dev).manual_seed(0)
    out = {"card": card(), "rows": a.rows, "dim": a.dim, "k": a.k, "cases": []}
    for dt in a.dtypes.split(","):
        tdt = {"f32": torch.float32, "f16": torch.float16}[dt]
        x = torch.randn(a.rows, a.dim, generator=g, device=dev, dtype=torch.float32).to(tdt)
        for q in [int(v) for v in a.probes.split(",")]:
            p = torch.randn(q, a.dim, generator=g, device=dev, dtype=torch.float64)
            phat = (p / p.norm(dim=1, keepdim=True)).float()
            s, r = ops.knn_topk(x, phat, a.k)                     # warm-up (module load, shape attributes)
            ms = event_ms(lambda: ops.knn_topk(x, phat, a.k), a.reps)
            ts, tr = torch_topk(x, phat, a.k)
            tms = event_ms(lambda: torch_topk(x, phat, a.k), max(1, a.reps // 2))
            esize = x.element_size()
            case = {"dtype": dt, "q": q, "kernel_ms": ms, "torch_fp32_ms": tms, "vs_torch": tms / ms,
                    "roofline": roofline(a.rows * a.dim * esize, 2 * a.rows * a.dim * q * TERMS[dt], ms / 1e3),
                    "agree_outside_tie_band": agreement(x, phat, r.cpu(), tr.cpu(), a.dim)}
            out["cases"].append(case)
            print(json.dumps(case), file=sys.stderr, flush=True)
        del x
    print(json.dumps(out))
    return out


if __name__ == "__main__":
    main()
