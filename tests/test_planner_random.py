"""Differential test of the planner: random DataStream programs (filter / with_columns / select / rename / join /
group-by) run through predicate push-down, projection pruning, edge-op folding, join role assignment, Bloom reduction
and the two-phase aggregate (on the numpy kernel shim), and step by step through pandas.  The two must return the
same relation."""
import numpy as np
import pandas as pd
import pyarrow as pa
import pytest
import torch

import cpu_shim
from quokka_b200 import expr as E

RTOL = 1e-9


@pytest.fixture
def qc(monkeypatch):
    cpu_shim.install(monkeypatch)
    import quokka_b200.df as D
    import quokka_b200.runtime as RT
    monkeypatch.setattr(D, "_default_device", lambda: torch.device("cpu"))
    monkeypatch.setattr(RT, "_default_device", lambda: torch.device("cpu"))
    from quokka_b200.df import QuokkaContext
    q = QuokkaContext()
    q.set_config("broadcast_rows", 10)              # shuffle-shaped joins (Bloom reduction included) even at this size
    return q


def _is_str(col) -> bool:
    return not pd.api.types.is_numeric_dtype(col)


def _tables(rng):
    na, nb = 400, 120
    a = pd.DataFrame({"k": rng.integers(0, 60, na), "x": rng.integers(0, 200, na) / 4.0, "y": rng.integers(-5, 6, na),
                      "s": rng.choice(["red", "green", "blue"], na), "d": (8000 + rng.integers(0, 900, na)).astype(np.int32)})
    b = pd.DataFrame({"k2": rng.permutation(np.arange(0, 120))[:nb] // 2, "z": rng.integers(0, 100, nb) / 2.0, "w": rng.integers(0, 4, nb),
                      "t": rng.choice(["N", "S"], nb), "y": rng.integers(0, 9, nb)})        # "y" clashes with the left table: suffix "_2"
    return a, b


def _third(rng):
    return pd.DataFrame({"k3": np.arange(-5, 12), "q": rng.integers(1, 9, 17) * 1.5, "u": rng.choice(["p", "q"], 17)})


def _arrow(df):
    cols = {}
    for c in df.columns:
        v = df[c].to_numpy()
        cols[c] = pa.array(v, pa.int32()).cast(pa.date32()) if c == "d" else pa.array(list(v) if _is_str(df[c]) else v)
    return pa.table(cols)


def _ev(node, df):
    """expr.Node over a pandas frame -> numpy (floats; booleans as 0/1), the semantics the kernels implement."""
    n = len(df)
    k = node.kind
    if k == "col":
        return df[node.value].to_numpy()
    if k in ("num", "date"):
        return np.full(n, float(node.value))
    if k == "un":
        v = _ev(node.args[0], df)
        return -v.astype(np.float64) if node.value == "neg" else (v == 0).astype(np.float64)
    if k == "func" and node.value == "case":
        c, x, y = (_ev(a, df) for a in node.args)
        return np.where(c != 0, x.astype(np.float64), y.astype(np.float64))
    a, b = node.args
    op = node.value
    if b.kind == "str":
        eq = df[a.value].to_numpy() == b.value
        return (eq if op == "=" else ~eq).astype(np.float64)
    x, y = _ev(a, df).astype(np.float64), _ev(b, df).astype(np.float64)
    if op in "+-*":
        return {"+": x + y, "-": x - y, "*": x * y}[op]
    if op in ("and", "or"):
        return ((x != 0) & (y != 0) if op == "and" else (x != 0) | (y != 0)).astype(np.float64)
    return {"<": x < y, "<=": x <= y, ">": x > y, ">=": x >= y, "=": x == y, "!=": x != y}[op].astype(np.float64)


class _Gen:
    def __init__(self, rng):
        self.rng = rng
        self.fresh = 0

    def name(self):
        self.fresh += 1
        return f"c{self.fresh}"

    def numeric(self, df):
        return [c for c in df.columns if not _is_str(df[c]) and c != "d"]

    def num_expr(self, df, depth=2):
        r, cols = self.rng, self.numeric(df)
        if depth == 0 or r.random() < 0.35:
            return str(r.choice(cols + [str(int(r.integers(-3, 7))), f"{r.integers(0, 40) / 4}"]))
        if r.random() < 0.85:
            return f"({self.num_expr(df, depth - 1)} {r.choice(['+', '-', '*'])} {self.num_expr(df, depth - 1)})"
        return f"(case when {self.pred(df, 0)} then {self.num_expr(df, depth - 1)} else {self.num_expr(df, depth - 1)} end)"

    def pred(self, df, depth=2):
        r = self.rng
        if depth == 0 or r.random() < 0.45:
            strs = [c for c in df.columns if _is_str(df[c])]
            k = r.integers(0, 4)
            if k == 0 and strs:
                c = r.choice(strs)
                return f"{c} {r.choice(['=', '<>'])} '{r.choice(list(df[c].unique()) + ['zz']) if len(df) else 'zz'}'"
            if k == 1 and "d" in df.columns:
                return f"d {r.choice(['<', '>='])} date '1992-0{r.integers(1, 9)}-15'"
            return f"{self.num_expr(df, 1)} {r.choice(['<', '<=', '>', '>=', '=', '<>'])} {self.num_expr(df, 1)}"
        if r.random() < 0.8:
            return f"({self.pred(df, depth - 1)} {r.choice(['and', 'or'])} {self.pred(df, depth - 1)})"
        return f"(not {self.pred(df, depth - 1)})"

    def step(self, stream, df):
        """One random unary operator applied to both representations."""
        r = self.rng
        k = r.integers(0, 4)
        if k == 0:
            p = self.pred(df)
            return stream.filter_sql(p), df[_ev(E.parse(p), df) != 0].reset_index(drop=True), f"filter({p})"
        if k == 1:
            e, n = self.num_expr(df), self.name()
            out = df.copy()
            out[n] = _ev(E.parse(e), df).astype(np.float64)
            return stream.with_columns_sql(f"{e} as {n}"), out, f"with({n}={e})"
        if k == 2 and len(df.columns) > 2:
            keep = [c for c in df.columns if r.random() < 0.7] or [df.columns[0]]
            return stream.select(keep), df[keep], f"select({keep})"
        if k == 3 and r.random() < 0.3 and len(df.columns) > 2:
            c = str(r.choice(list(df.columns)))
            return stream.drop([c]), df.drop(columns=[c]), f"drop({c})"
        if k == 3 and r.random() < 0.3 and self.numeric(df):
            c = str(r.choice(self.numeric(df)))
            lo, hi = sorted(float(v) for v in r.integers(-4, 60, 2))
            out = df.copy()
            out[c] = np.clip(out[c].to_numpy(dtype=np.float64), lo, hi)
            return stream.clip({c: (lo, hi)}), out, f"clip({c},{lo},{hi})"
        if k == 3 and r.random() < 0.3 and self.numeric(df):
            keep = [c for c in df.columns if r.random() < 0.6] or [df.columns[0]]
            e, n = self.num_expr(df), self.name()
            out = df[keep].copy()
            out[n] = _ev(E.parse(e), df).astype(np.float64)
            return stream.transform_sql(", ".join(keep) + f", {e} as {n}"), out, f"transform_sql({keep}, {n}={e})"
        c, n = r.choice(list(df.columns)), self.name()
        return stream.rename({c: n}), df.rename(columns={c: n}), f"rename({c}->{n})"


def _same_relation(got: pa.Table, exp: pd.DataFrame, trace, nulls=False):
    assert sorted(got.column_names) == sorted(exp.columns), trace
    assert got.num_rows == len(exp), (got.num_rows, len(exp), trace)
    if not len(exp):
        return
    g = got.to_pandas()[list(exp.columns)]
    for c in exp.columns:                           # a date32 column comes back as dates: days since the epoch, like the frame
        if not _is_str(exp[c]) and not pd.api.types.is_numeric_dtype(g[c]):
            import datetime
            days = pd.Series([(v - datetime.date(1970, 1, 1)).days if isinstance(v, datetime.date) else np.nan for v in g[c]], index=g.index)
            g[c] = days if days.isna().any() else days.astype(np.int64)
    if nulls:                                       # unmatched rows of a left join: NULL on both sides -> one sentinel
        exp = exp.copy()
        for c in exp.columns:
            if _is_str(exp[c]):
                g[c], exp[c] = g[c].astype(object).where(g[c].notna(), "<null>"), exp[c].astype(object).where(exp[c].notna(), "<null>")
            else:
                g[c], exp[c] = g[c].astype(np.float64).fillna(-12345.0), exp[c].astype(np.float64).fillna(-12345.0)
    for c in exp.columns:
        if _is_str(exp[c]):
            g[c], exp[c] = g[c].astype(str), exp[c].astype(str)
    # order rows canonically on every column (values rounded for the sort only)
    key = lambda d: d.assign(**{c: d[c].round(6) for c in d.columns if pd.api.types.is_float_dtype(d[c])})
    gi = key(g).sort_values(list(exp.columns), kind="stable").index
    ei = key(exp).sort_values(list(exp.columns), kind="stable").index
    g, e = g.loc[gi].reset_index(drop=True), exp.loc[ei].reset_index(drop=True)
    for c in exp.columns:
        if pd.api.types.is_numeric_dtype(e[c]) and pd.api.types.is_numeric_dtype(g[c]):
            np.testing.assert_allclose(g[c].to_numpy(dtype=np.float64), e[c].to_numpy(dtype=np.float64), rtol=RTOL, atol=1e-9, err_msg=str(trace))
        else:
            assert list(g[c]) == list(e[c]), (c, trace)


@pytest.mark.parametrize("seed", [int(x) for x in __import__("os").environ.get("QK_PLANNER_SEEDS", "2025,7").split(",")])
def test_random_programs_agree_with_pandas(qc, seed):
    if seed % 2:                                    # odd seeds: sources arrive in many small batches (state across execute() calls,
        qc.set_config("chunk_rows", 33)             # dictionaries that grow from batch to batch)
    run_random_programs(qc, seed, int(__import__("os").environ.get("QK_PLANNER_TRIALS", "100")))


def run_random_programs(qc, seed, trials, parquet_dir=None):
    """Also driven by tests/test_dist_gloo.py on two ranks: every rank draws the same programs from the same seed.
    With `parquet_dir` the left input is a Parquet file sorted on `k` with small row groups, read by the host reader or
    (every other trial) decoded on the device: the planner's pruning hints then skip row groups under random predicates."""
    rng = np.random.default_rng(seed)
    a_df, b_df = _tables(rng)
    if parquet_dir is not None:
        import os
        import pyarrow.parquet as pq
        a_df = a_df.sort_values(["k", "d"], kind="stable").reset_index(drop=True)
        a_path = os.path.join(str(parquet_dir), f"a_{seed}.parquet")
        pq.write_table(_arrow(a_df), a_path, row_group_size=40, compression=["snappy", "zstd", None][seed % 3])
    a_tab, b_tab = _arrow(a_df), _arrow(b_df)
    c_df = _third(rng)
    c_tab = _arrow(c_df)
    for trial in range(trials):
        gen = _Gen(rng)
        trace = [f"trial {trial}"]
        if parquet_dir is not None:
            qc.set_config("device_parquet", bool(trial % 2))
            s, df = qc.read_parquet(a_path), a_df.copy()
            trace.append(f"parquet(device={bool(trial % 2)})")
        else:
            s, df = qc.from_arrow(a_tab), a_df.copy()
        df["d"] = df["d"].astype(np.int64)
        for _ in range(rng.integers(0, 3)):
            s, df, t = gen.step(s, df)
            trace.append(t)
        if rng.random() < 0.7 and len(gen.numeric(df)) > 0:
            r, rdf = qc.from_arrow(b_tab), b_df.copy()
            for _ in range(rng.integers(0, 2)):
                r, rdf, t = gen.step(r, rdf)
                trace.append("right:" + t)
            lk = [c for c in df.columns if pd.api.types.is_integer_dtype(df[c]) and c != "d"]
            rk = [c for c in rdf.columns if pd.api.types.is_integer_dtype(rdf[c])]
            if rng.random() < 0.15:                             # a self join: the same source twice, the right side renamed
                r, rdf = qc.from_arrow(a_tab), a_df.copy()
                rdf["d"] = rdf["d"].astype(np.int64)
                ren = {c: c + "_r" for c in rdf.columns}
                r, rdf = r.rename(ren).select(["k_r", "x_r", "s_r"]), rdf.rename(columns=ren)[["k_r", "x_r", "s_r"]]
                trace.append("right:self")
                rk = ["k_r"]
            if lk and rk:
                lo, ro, how = rng.choice(lk), rng.choice(rk), rng.choice(["inner", "semi", "anti", "left"])
                trace.append(f"join({how} {lo}={ro})")
                s = s.join(r, left_on=lo, right_on=ro, how=how)
                if how == "inner":
                    rr = rdf.rename(columns={ro: "__rk"})
                    df = df.merge(rr, left_on=lo, right_on="__rk", how="inner", suffixes=("", "_2")).drop(columns=["__rk"])   # right key dropped
                elif how == "left":
                    # the build side must be unique on its key for pandas and the engine to agree on row multiplicity -- it
                    # is not in general, so compare multisets: a left join keeps every probe row at least once
                    rr = rdf.rename(columns={ro: "__rk"})
                    df = df.merge(rr, left_on=lo, right_on="__rk", how="left", suffixes=("", "_2")).drop(columns=["__rk"])
                    trace.append("left->collect")
                    if len(rdf) == 0:
                        # the reference's executor emits NOTHING for a left join whose build side is empty
                        # (pyquokka/executors/sql_executors.py:362-366; SURVEY.md Appendix A-5) -- kept, quirk and all
                        assert s.collect().num_rows == 0, trace
                        continue
                    _same_relation(s.collect(), df.reset_index(drop=True), trace, nulls=True)
                    continue
                else:
                    hit = df[lo].isin(rdf[ro])
                    df = df[hit if how == "semi" else ~hit]
                df = df.reset_index(drop=True)
                for _ in range(rng.integers(0, 3)):
                    s, df, t = gen.step(s, df)
                    trace.append(t)
        ints = [c for c in df.columns if pd.api.types.is_integer_dtype(df[c]) and c != "d"]
        if rng.random() < 0.3 and ints:                      # a second join, against a small third table
            lo = rng.choice(ints)
            trace.append(f"join2(inner {lo}=k3)")
            s = s.join(qc.from_arrow(c_tab), left_on=lo, right_on="k3")
            df = df.merge(c_df, left_on=lo, right_on="k3", how="inner").drop(columns=["k3"]).reset_index(drop=True)
            for _ in range(rng.integers(0, 2)):
                s, df, t = gen.step(s, df)
                trace.append(t)
        assert list(s.schema) == list(df.columns), trace
        end = rng.random()
        if end < 0.15:
            keys = [c for c in df.columns if (_is_str(df[c]) or pd.api.types.is_integer_dtype(df[c])) and c != "d"][:2]
            if keys:
                trace.append(f"distinct({keys})")
                _same_relation(s.distinct(keys).collect(), df[keys].drop_duplicates().reset_index(drop=True), trace)
                continue
        elif end < 0.3 and gen.numeric(df) and len(df) > 5:
            v = rng.choice(gen.numeric(df))
            trace.append(f"top_k({v}, 5)")
            got = s.top_k(v, 5, descending=True).collect()
            assert got.num_rows == 5 and got.column_names == list(df.columns), trace
            np.testing.assert_allclose(np.sort(got[v].to_numpy().astype(np.float64)), np.sort(df[v].to_numpy(dtype=np.float64))[-5:], rtol=RTOL, err_msg=str(trace))
            continue
        elif end < 0.4 and len(df):
            c = str(rng.choice([c for c in df.columns if c != "d" and (_is_str(df[c]) or pd.api.types.is_integer_dtype(df[c]))] or [df.columns[0]]))
            if c != "d" and not pd.api.types.is_float_dtype(df[c]):
                trace.append(f"count_distinct({c})")
                got = s.count_distinct(c).collect()
                assert int(got[got.column_names[0]][0].as_py()) == df[c].nunique(), trace
                continue
        elif end < 0.5 and gen.numeric(df) and len(df):
            v = str(rng.choice(gen.numeric(df)))
            trace.append(f"agg dict({v})")
            got = s.agg({v: ["sum", "max"], "*": "count"}).collect()
            assert got.num_rows == 1, trace
            np.testing.assert_allclose([got[f"{v}_sum"][0].as_py(), got[f"{v}_max"][0].as_py(), got["count"][0].as_py()],
                                       [df[v].sum(), df[v].max(), len(df)], rtol=RTOL, err_msg=str(trace))
            continue
        if rng.random() < 0.5 and gen.numeric(df):
            keys = [c for c in df.columns if (_is_str(df[c]) or pd.api.types.is_integer_dtype(df[c])) and c != "d" and rng.random() < 0.4][:2]
            v = rng.choice(gen.numeric(df))
            trace.append(f"groupby({keys}) on {v}")
            sql = f"sum({v}) as s_, min({v}) as lo_, max({v}) as hi_, count(*) as n_, avg({v}) as a_"
            if rng.random() < 0.3:                           # expressions over aggregates (Q14's ratio of sums, Q1's averages)
                sql2 = f"sum({v}) / count(*) as r1_, max({v}) - min({v}) as r2_, 100.0 * sum({v} * 2) / (1 + sum({v} * {v})) as r3_"
                got2 = (s.groupby(keys).agg_sql(sql2) if keys else s.agg_sql(sql2)).collect()
                if len(df):
                    gb = df.assign(__v2=df[v] * 2.0, __vv=df[v].astype(np.float64) * df[v]).groupby(keys, as_index=False) if keys else None
                    if keys:
                        e2 = gb.agg(__s=(v, "sum"), __n=(v, "size"), __hi=(v, "max"), __lo=(v, "min"), __s2=("__v2", "sum"), __svv=("__vv", "sum"))
                    else:
                        e2 = pd.DataFrame({"__s": [df[v].sum()], "__n": [len(df)], "__hi": [df[v].max()], "__lo": [df[v].min()],
                                           "__s2": [(df[v] * 2.0).sum()], "__svv": [(df[v].astype(np.float64) * df[v]).sum()]})
                    e2 = e2.assign(r1_=e2.__getitem__("__s") / e2["__n"], r2_=(e2["__hi"] - e2["__lo"]).astype(np.float64),
                                   r3_=100.0 * e2["__s2"] / (1 + e2["__svv"]))[keys + ["r1_", "r2_", "r3_"]]
                    trace.append("ratios")
                    _same_relation(got2, e2, trace)
            got = (s.groupby(keys).agg_sql(sql) if keys else s.agg_sql(sql)).collect()
            if keys:
                exp = df.groupby(keys, as_index=False).agg(s_=(v, "sum"), lo_=(v, "min"), hi_=(v, "max"), n_=(v, "size"), a_=(v, "mean"))
            elif len(df):
                exp = pd.DataFrame({"s_": [df[v].sum()], "lo_": [df[v].min()], "hi_": [df[v].max()], "n_": [len(df)], "a_": [df[v].mean()]})
            else:
                exp = pd.DataFrame({c: [] for c in ("s_", "lo_", "hi_", "n_", "a_")})
            if got.num_rows == 0 and not len(exp):
                continue
            _same_relation(got, exp.astype({c: np.float64 for c in ("s_", "lo_", "hi_", "n_", "a_")}), trace)
            if keys and rng.random() < 0.5:                  # HAVING: a filter over the aggregate's output
                trace.append("having(n_ > 1 and s_ >= lo_)")
                h = s.groupby(keys).agg_sql(sql).filter_sql("n_ > 1 and s_ >= lo_").collect()
                e2 = exp[(exp.n_ > 1) & (exp.s_ >= exp.lo_)].reset_index(drop=True)
                if h.num_rows or len(e2):
                    _same_relation(h, e2.astype({c: np.float64 for c in ("s_", "lo_", "hi_", "n_", "a_")}), trace)
        else:
            _same_relation(s.collect(), df.copy(), trace)


def test_random_programs_over_parquet(qc, tmp_path):
    run_random_programs(qc, 77, 80, tmp_path)
    run_random_programs(qc, 78, 40, tmp_path)


def run_random_asof(qc, seed, trials=12):
    """Streaming as-of joins (OrderedStream.join_asof -> SortedAsofExecutor) on random time-sorted inputs cut into small
    batches -- so that trades wait in the executor's state for newer quotes, across many execute() calls -- against
    pandas.merge_asof (backward, by symbol, exact matches allowed, the last of equal-time quotes wins)."""
    rng = np.random.default_rng(seed)
    for trial in range(trials):
        nt, nq, nsym = int(rng.integers(1, 400)), int(rng.integers(1, 900)), int(rng.integers(1, 6))
        span = int(rng.integers(5, 2000))                    # small spans force many equal timestamps
        trades = pd.DataFrame({"time": np.sort(rng.integers(0, span, nt)).astype(np.int64), "symbol": rng.choice([f"S{i}" for i in range(nsym)], nt),
                               "size": rng.integers(1, 100, nt).astype(np.float64)})
        quotes = pd.DataFrame({"time": np.sort(rng.integers(0, span, nq)).astype(np.int64), "symbol": rng.choice([f"S{i}" for i in range(nsym + 1)], nq),
                               "bid": rng.integers(1, 1000, nq) / 8.0, "iq": np.arange(nq, dtype=np.int64)})
        qc.set_config("chunk_rows", int(rng.integers(7, 200)))
        try:
            t = qc.from_arrow_sorted(pa.Table.from_pandas(trades, preserve_index=False), "time")
            q = qc.from_arrow_sorted(pa.Table.from_pandas(quotes, preserve_index=False), "time")
            got = t.join_asof(q, on="time", by="symbol").collect().to_pandas()
        finally:
            qc.set_config("chunk_rows", 1 << 26)
        exp = pd.merge_asof(trades.reset_index(names="row"), quotes, on="time", by="symbol", direction="backward", allow_exact_matches=True)
        assert len(got) == nt and sorted(got.columns) == sorted(["time", "symbol", "size", "bid", "iq"]), (seed, trial)
        # equal (time, symbol, size) trades are interchangeable: compare as multisets of full rows
        key = ["time", "symbol", "size", "iq", "bid"]
        g = got[key].fillna(-1.0).sort_values(key).reset_index(drop=True)
        e = exp[key].fillna(-1.0).sort_values(key).reset_index(drop=True)
        assert g["symbol"].astype(str).tolist() == e["symbol"].astype(str).tolist(), (seed, trial)
        for c in ("time", "size", "iq", "bid"):
            assert np.array_equal(g[c].to_numpy(dtype=np.float64), e[c].to_numpy(dtype=np.float64)), (seed, trial, c)


def run_asof_rank_shards(qc, seed, trials=14):
    """The multi-rank as-of join over TIME RANGES (SortedAsofExecutor._join_time_ranges): every rank passes its own contiguous
    slice of the two sorted streams, cut independently -- so trades sit on the "wrong" side of a quote boundary, ranks have no
    quotes, no trades, or nothing at all, and equal timestamps straddle the cuts -- and every rank must collect the global join."""
    from quokka_b200 import runtime
    from quokka_b200.columns import DeviceTable
    w, me = runtime.world_size(), runtime.rank()
    rng = np.random.default_rng(seed)                      # the same draws on every rank
    for trial in range(trials):
        nt, nq, nsym = int(rng.integers(0, 300)), int(rng.integers(1, 600)), int(rng.integers(1, 5))
        span = int(rng.integers(3, 500))
        trades = pd.DataFrame({"time": np.sort(rng.integers(0, span, nt)).astype(np.int64), "symbol": rng.integers(0, nsym, nt).astype(np.int32),
                               "size": rng.integers(1, 100, nt).astype(np.float64)})
        quotes = pd.DataFrame({"time": np.sort(rng.integers(0, span, nq)).astype(np.int64), "symbol": rng.integers(0, nsym + 1, nq).astype(np.int32),
                               "iq": np.arange(nq, dtype=np.int64)})
        # every symbol has a quote at the very start: with the reference's hash shuffle a rank that received trades but no quote
        # at all cannot know the quote columns (the reference's executor fails there too); the time-range join handles that case
        # and gets it from the cuts below (ranks without quotes)
        first = pd.DataFrame({"time": np.zeros(nsym + 1, dtype=np.int64), "symbol": np.arange(nsym + 1, dtype=np.int32), "iq": -1 - np.arange(nsym + 1, dtype=np.int64)})
        quotes = pd.concat([first, quotes], ignore_index=True)
        nq = len(quotes)
        if trial % 3 == 2:      # a string payload column: every rank's shard has its own dictionary, the carried rows another one
            quotes["venue"] = rng.choice(["ARCA", "BATS", "IEX", "NYSE", "NSDQ"], nq)
        style = trial % 4                                   # 0: random cuts, 1: all quotes on the last rank, 2: all trades on rank 0, 3: rank 0 empty
        def cuts(n, kind):
            if style == 1 and kind == "q":
                return [0] * w + [n]
            if style == 2 and kind == "t":
                return [0] + [n] * w
            c = sorted(int(x) for x in rng.integers(0, n + 1, w - 1))
            if style == 3:
                c[0] = 0
            return [0] + c + [n]
        ct, cq = cuts(nt, "t"), cuts(nq, "q")
        mine_t = trades.iloc[ct[me]:ct[me + 1]]
        mine_q = quotes.iloc[cq[me]:cq[me + 1]]
        t = qc.from_device(DeviceTable.from_arrow(pa.Table.from_pandas(mine_t, preserve_index=False)), sorted_by="time")
        q = qc.from_device(DeviceTable.from_arrow(pa.Table.from_pandas(mine_q, preserve_index=False)), sorted_by="time")
        got = t.join_asof(q, on="time", by="symbol").collect().to_pandas()
        exp = pd.merge_asof(trades, quotes, on="time", by="symbol", direction="backward", allow_exact_matches=True)
        assert len(got) == nt, (seed, trial, len(got), nt)
        if nt == 0:
            continue
        key = ["time", "symbol", "size", "iq"]
        extra = ["venue"] if "venue" in quotes.columns else []
        g = got[key + extra].fillna(-1.0).sort_values(key).reset_index(drop=True)
        e = exp[key + extra].fillna(-1.0).sort_values(key).reset_index(drop=True)
        for c in key:
            assert np.array_equal(g[c].to_numpy(dtype=np.float64), e[c].to_numpy(dtype=np.float64)), (seed, trial, style, c)
        for c in extra:
            assert g[c].astype(str).tolist() == e[c].astype(str).tolist(), (seed, trial, style, c)


def test_random_asof_joins_agree_with_pandas(qc):
    run_random_asof(qc, 5, 25)
