"""Regenerates tests/golden/asof_strategy2.npz from the reference's own fixture apps/time-series/test_trade2.csv x
test_quote2.csv (26 duplicate (time, symbol) quote pairs): the right-row index pandas.merge_asof(by=symbol) matches for
direction "forward" and "nearest", without a tolerance and with TOLERANCE.  The tests read only the committed .npz file.

usage: python tests/golden/make_golden_asof_strategy.py <reference checkout>"""
import os
import sys

import numpy as np
import pandas as pd

REF = sys.argv[1] if len(sys.argv) > 1 else "."
OUT = os.path.dirname(os.path.abspath(__file__))
TOLERANCE = 40


def main():
    t = pd.read_csv(f"{REF}/apps/time-series/test_trade2.csv")
    q = pd.read_csv(f"{REF}/apps/time-series/test_quote2.csv")
    syms = sorted(set(t.symbol) | set(q.symbol))
    code = {s: i for i, s in enumerate(syms)}
    t["sym"] = t.symbol.map(code).astype(np.int32)
    q["sym"] = q.symbol.map(code).astype(np.int32)
    q["iq"] = np.arange(len(q))
    out = dict(t_time=t.time.to_numpy(np.int64), t_sym=t.sym.to_numpy(np.int32), q_time=q.time.to_numpy(np.int64),
               q_sym=q.sym.to_numpy(np.int32), tolerance=TOLERANCE)
    for direction in ("forward", "nearest"):
        for tol, tag in ((None, ""), (TOLERANCE, "_tol")):
            m = pd.merge_asof(t, q[["time", "sym", "iq"]], on="time", by="sym", direction=direction, tolerance=tol)
            out[f"ridx_{direction}{tag}"] = m.iq.fillna(-1).to_numpy(np.int64)
            print(direction, tol, int((out[f"ridx_{direction}{tag}"] >= 0).sum()), "of", len(t), "matched")
    dup = q.duplicated(["time", "sym"]).sum()
    print("duplicate (time, symbol) quote pairs:", int(dup))
    np.savez_compressed(f"{OUT}/asof_strategy2.npz", **out)


if __name__ == "__main__":
    main()
