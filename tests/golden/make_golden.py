"""Regenerates tests/golden/*.npz from the reference's own fixtures:

  python tests/golden/make_golden.py <checkout of marsupialtail/quokka @ 1caf62e>

The tests read only the committed .npz files; they never need the reference itself.

  join_ab.npz   <- apps/graph_api/tutorials/a.csv, b.csv (the lesson2.1.py:57-68 join self-check;
                   expected pairs from pandas.merge, the engine that script compares against)
  asof_*.npz    <- apps/time-series/test_trade{,1,2}.csv x test_quote{,1,2}.csv (asof_join.py:6-18;
                   expected right-row index from pandas.merge_asof(direction="backward", by=symbol),
                   which agrees with the Polars call the script uses as its own reference)
"""
import os
import sys
import numpy as np
import pandas as pd

REF = sys.argv[1] if len(sys.argv) > 1 else "."
OUT = os.path.dirname(os.path.abspath(__file__))


def join_ab():
    a = pd.read_csv(f"{REF}/apps/graph_api/tutorials/a.csv")
    b = pd.read_csv(f"{REF}/apps/graph_api/tutorials/b.csv")
    a["ia"] = np.arange(len(a)); b["ib"] = np.arange(len(b))
    inner = a.merge(b, left_on="key_a", right_on="key_b", how="inner")
    left = a.merge(b, left_on="key_a", right_on="key_b", how="left")
    semi = a[a.key_a.isin(b.key_b)]
    anti = a[~a.key_a.isin(b.key_b)]
    np.savez_compressed(f"{OUT}/join_ab.npz",
        key_a=a.key_a.to_numpy(np.int64), val1_a=a.val1_a.to_numpy(), val2_a=a.val2_a.to_numpy(),
        key_b=b.key_b.to_numpy(np.int64), val1_b=b.val1_b.to_numpy(), val2_b=b.val2_b.to_numpy(),
        inner_ia=inner.ia.to_numpy(np.int64), inner_ib=inner.ib.to_numpy(np.int64),
        n_inner=len(inner), n_left=len(left), n_semi=len(semi), n_anti=len(anti),
        dot_val1=float((inner.val1_a * inner.val1_b).sum()))
    print("join_ab", len(inner), len(left), len(semi), len(anti))


def asof(tag):
    t = pd.read_csv(f"{REF}/apps/time-series/test_trade{tag}.csv")
    q = pd.read_csv(f"{REF}/apps/time-series/test_quote{tag}.csv")
    syms = sorted(set(t.symbol) | set(q.symbol))
    code = {s: i for i, s in enumerate(syms)}
    t["sym"] = t.symbol.map(code).astype(np.int32); q["sym"] = q.symbol.map(code).astype(np.int32)
    q["iq"] = np.arange(len(q))
    m = pd.merge_asof(t, q[["time", "sym", "iq", "asize"]], on="time", by="sym", direction="backward")
    ridx = m.iq.fillna(-1).to_numpy(np.int64)
    matched = ridx >= 0
    np.savez_compressed(f"{OUT}/asof{tag or '0'}.npz",
        t_time=t.time.to_numpy(np.int64), t_sym=t.sym.to_numpy(np.int32), t_size=t["size"].to_numpy(),
        q_time=q.time.to_numpy(np.int64), q_sym=q.sym.to_numpy(np.int32), q_asize=q.asize.to_numpy(),
        ridx=ridx, n_matched=int(matched.sum()), sum_size=float(t["size"].to_numpy()[matched].sum()),
        sum_asize100=int(np.rint(q.asize.to_numpy()[ridx[matched]] * 100).sum()))
    print("asof", tag, len(t), int(matched.sum()))


def asof_result():
    """apps/time-series/result.csv: an output the reference itself produced for asof_join.py on test_trade2 / test_quote2
    (trades.join_asof(quotes, on=time, by=symbol).drop_nulls()) -- the one place the reference holds a golden RESULT
    for an executor.  It is a partial dump (2 996 of the 3 995 matched trades).  2 995 of its rows equal
    pandas.merge_asof / Polars join_asof on the same files; ONE row (trade time 48589, ZUMZ) carries the quote of an
    earlier batch boundary instead of the newest quote (SURVEY.md section 4: the streaming executor's known
    batch-boundary defect), so it is recorded separately as the documented exception."""
    res = pd.read_csv(f"{REF}/apps/time-series/result.csv")
    t = pd.read_csv(f"{REF}/apps/time-series/test_trade2.csv")
    q = pd.read_csv(f"{REF}/apps/time-series/test_quote2.csv")
    exp = pd.merge_asof(t, q, on="time", by="symbol", direction="backward").dropna()
    pay = [c for c in res.columns if c not in ("time", "symbol")]
    from collections import Counter
    rows = lambda df: [tuple(r) for r in df[list(res.columns)].round(9).astype(str).values.tolist()]
    have = Counter(rows(exp))
    same = np.zeros(len(res), bool)
    for i, r in enumerate(rows(res)):                 # multiset containment: every result.csv row must be a row of the join
        if have[r] > 0:
            have[r] -= 1
            same[i] = True
    assert int((~same).sum()) == 1, int((~same).sum())
    syms = sorted(set(t.symbol) | set(q.symbol))
    code = {s: i for i, s in enumerate(syms)}
    good = res[same]
    bad = res[~same]
    np.savez_compressed(f"{OUT}/asof_result2.npz",
        time=good.time.to_numpy(np.int64), sym=good.symbol.map(code).to_numpy(np.int32),
        **{c: good[c].to_numpy() for c in pay},
        bad_time=bad.time.to_numpy(np.int64), bad_sym=bad.symbol.map(code).to_numpy(np.int32),
        symbols=np.array(syms),
        # the inputs in full (the asof*.npz fixtures keep only the columns the checksum needs)
        **{"in_t_" + c: (t[c].map(code).to_numpy(np.int32) if c == "symbol" else t[c].to_numpy()) for c in t.columns},
        **{"in_q_" + c: (q[c].map(code).to_numpy(np.int32) if c == "symbol" else q[c].to_numpy()) for c in q.columns})
    print("asof_result2", len(good), "rows equal the correct join,", len(bad), "documented exception")


if __name__ == "__main__":
    asof_result()
    join_ab()
    for tag in ("", "1", "2"):
        asof(tag)
