"""The time-series window kernels (csrc/window.cu) against the vectorised references of oracle/relops.py, the windowed and as-of
API at scale, and key counts above the shared-memory limits: the CODE partition past 16 384 parts (csrc/partition.cu), the
as-of merge kernel's 40 960-key table and the search path that takes over above it (csrc/asof.cu).

Inputs of the window kernels are built in numpy (sorted by key and time, segments from np.bincount), so these tests do not
depend on the partition kernel.  Two value columns:
  exact    integer multiples of 2^-4 with |v| <= 2^20: every partial sum is exact in fp64, so SUM / MIN / MAX / COUNT must
           match bit for bit and AVG too (one rounding of an exact quotient);
  general  magnitudes 1e-3 .. 1e8, both signs: SUM within the bound of sequential summation, (w - 1) * 2^-53 * sum|v| over a
           window of w rows, of the exact sum (relops.range_sum_exact); MIN / MAX bit for bit."""
import datetime
import types

import numpy as np
import pytest
import torch

from oracle import relops as R

pytestmark = pytest.mark.gpu

U = 2.0 ** -53


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def host(t):
    return t.cpu().numpy()


@pytest.fixture(scope="module")
def qb():
    from quokka_b200 import _lib, ops, synth
    _lib.lib()
    return types.SimpleNamespace(L=_lib, ops=ops, synth=synth)


def exact_col(rng, n):
    return rng.integers(-2 ** 24, 2 ** 24 + 1, n).astype(np.float64) / 16.0


def general_col(rng, n):
    return 10.0 ** rng.uniform(-3, 8, n) * np.where(rng.random(n) < 0.5, -1.0, 1.0)


def segmented(time, by, n_by):
    """Rows in key-segmented order (by key, then time, then input order) and seg[n_by + 1] from the key counts."""
    order = np.lexsort((time, by))
    seg = np.concatenate([[0], np.cumsum(np.bincount(by, minlength=n_by))]).astype(np.int64)
    return order, seg


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.int64)


def check_sum(got, v, lo, hi, what):
    """got[j] = a sum of v[lo[j]:hi[j]] in some order: within (w - 1) * 2^-53 * sum|v| of the exact sum (plus the
    reference's own long-double rounding)."""
    exact = R.range_sum_exact(v, lo, hi)
    s_abs = R.range_sum_exact(np.abs(v), lo, hi)
    w = (hi - lo).astype(np.longdouble)
    err = np.abs(got.astype(np.longdouble) - exact)
    tol = (w - 1) * np.longdouble(U) * s_abs + np.longdouble(2.0 ** -62) * s_abs
    bad = np.flatnonzero(err > tol)
    assert not len(bad), (what, bad[:5], got[bad[:5]], exact[bad[:5]], tol[bad[:5]])


def check_avg(got, v, lo, hi, what):
    exact = R.range_sum_exact(v, lo, hi)
    s_abs = R.range_sum_exact(np.abs(v), lo, hi)
    w = (hi - lo).astype(np.longdouble)
    err = np.abs(got.astype(np.longdouble) - exact / w)
    tol = ((w - 1) * np.longdouble(U) * s_abs * (1 + np.longdouble(U)) + np.longdouble(U + 2.0 ** -62) * s_abs) / w
    bad = np.flatnonzero(err > tol)
    assert not len(bad), (what, bad[:5], got[bad[:5]], (exact / w)[bad[:5]])


def check_agg(op, got, v, exact_vals, lo, hi, what):
    """One window aggregate against the references: bit for bit where the column is exact or the op is MIN / MAX / COUNT."""
    if op == "count":
        assert np.array_equal(got, (hi - lo).astype(np.float64)), what
    elif op in ("min", "max") or exact_vals:
        exp = R.range_aggregate(op, v, lo, hi)
        bad = np.flatnonzero(bits(got) != bits(exp))
        assert not len(bad), (what, op, bad[:5], got[bad[:5]], exp[bad[:5]])
    elif op == "sum":
        check_sum(got, v, lo, hi, what)
    else:
        check_avg(got, v, lo, hi, what)


def draw_keys(rng, n, nkeys):
    """Key codes in [0, nkeys) with every fifth key (1, 6, 11, ...) left without rows."""
    live = np.arange(nkeys)
    if nkeys > 1:
        live = live[live % 5 != 1]
    return live[rng.integers(0, len(live), n)].astype(np.int32)


def draw_times(rng, n, nkeys, kind):
    if kind == "tiny":                                    # heavy ties: a few distinct times per key
        return np.sort(rng.integers(0, max(2, n // (40 * nkeys)), n)).astype(np.int64)
    if kind == "neg":
        return np.sort(rng.integers(-10 * n - 5, 0, n)).astype(np.int64)
    big = np.int64(2 ** 62)                               # two clusters near -2^62 and +2^62
    t = np.where(rng.random(n) < 0.5, -big + rng.integers(0, 1000, n), big - rng.integers(0, 1000, n))
    return np.sort(t).astype(np.int64)


# ------------------------------------------------------------------ sliding windows
_OPS = ["sum", "min", "max", "count", "avg"]


def _win_specs(qb):
    """16 outputs over 8 value columns (even: exact, odd: general); every column feeds two outputs."""
    code = {"sum": qb.L.WIN_SUM, "min": qb.L.WIN_MIN, "max": qb.L.WIN_MAX, "count": qb.L.WIN_COUNT, "avg": qb.L.WIN_AVG}
    names = [(_OPS[i % 5], (3 * i) % 8) for i in range(16)]
    return names, [(code[op], src) for op, src in names]


@pytest.mark.parametrize("n,nkeys,kind,size", [
    (1, 1, "tiny", 1),
    (255, 3, "tiny", 1), (256, 3, "neg", 5), (257, 1, "huge", 2 ** 62), (257, 3, "huge", 1),
    (2049, 3, "tiny", 2), (2049, 1, "neg", 10 ** 9), (2049, 8000, "neg", 10 ** 9),
    (100_003, 1, "tiny", 1), (100_003, 3, "neg", 300), (100_003, 8000, "huge", 2 ** 62), (100_003, 8000, "tiny", 3),
    (100_003, 8000, "neg", 10 ** 9)])
def test_window_sliding_kernel(qb, n, nkeys, kind, size):
    """Every row aggregates its key's rows with time in (t - size, t]: size 1 is exactly the row's tie group, sizes larger
    than the time span take the whole segment up to the row's ties, and keys without rows sit between keys with rows."""
    rng = np.random.default_rng(n * 7 + nkeys + len(kind))
    time, by = draw_times(rng, n, nkeys, kind), draw_keys(rng, n, nkeys)
    order, seg = segmented(time, by, nkeys)
    ts, bs = time[order], by[order]
    vals = [(exact_col if c % 2 == 0 else general_col)(rng, n) for c in range(8)]
    names, specs = _win_specs(qb)
    outs = qb.ops.window_sliding(dev(ts), dev(bs), dev(seg), nkeys, size, [dev(v) for v in vals], specs)
    ro, lo, hi = R.sliding_window_ranges(ts, bs, size)
    assert np.array_equal(ro, np.arange(n))                          # the inputs are already in the reference's order
    assert np.all(hi > np.arange(n)) and np.all(lo <= np.arange(n))
    for (op, src), o in zip(names, outs):
        check_agg(op, host(o), vals[src], src % 2 == 0, lo, hi, (op, src))


# ------------------------------------------------------------------ hopping windows
def hop_rule(ts, bs, seg, size, hop):
    """The expansion rule: row i, slot q -> k = floor(t / hop) - q; the slot is used when floor((t - size) / hop) < k and
    k * hop is not before the key's first time truncated to hop."""
    slots = -(-size // hop)
    n = len(ts)
    first = (ts[seg[bs]] // hop) * hop if n else np.zeros(0, np.int64)
    k = (ts // hop)[:, None] - np.arange(slots, dtype=np.int64)[None, :]
    valid = (k > ((ts - size) // hop)[:, None]) & (k * hop >= first[:, None])
    return (k * hop).reshape(-1), np.repeat(bs, slots), np.where(valid, np.arange(n)[:, None], -1).reshape(-1).astype(np.int32)


@pytest.mark.parametrize("size,hop", [(3000, 1000), (2500, 1000), (300, 1000), (1000, 1), (1000, 1000)])
@pytest.mark.parametrize("neg", [False, True])
def test_window_hop_expand_and_aggregate(qb, size, hop, neg):
    """Slot by slot against the rule, then the whole hopping aggregate (expand -> compaction -> gather -> hash aggregate, as
    HoppingWindowExecutor.done runs it) against the reference: 2500 / 1000 has a partial last slot, 300 / 1000 leaves rows
    in no window, 1000 / 1 gives every row a thousand windows."""
    L, ops = qb.L, qb.ops
    rng = np.random.default_rng(size + hop + neg)
    n, nkeys = (5_000 if hop == 1 else 200_003), 300
    time = np.sort(rng.integers(0, 30 * n, n)).astype(np.int64)
    if neg:
        time = time - 40 * n - 7
    by = draw_keys(rng, n, nkeys)
    order, seg = segmented(time, by, nkeys)
    ts, bs = time[order], by[order]
    ve, vg = exact_col(rng, n), general_col(rng, n)
    wstart, key, src = ops.window_hop_expand(dev(ts), dev(bs), dev(seg), nkeys, size, hop)
    ew, ek, es = hop_rule(ts, bs, seg, size, hop)
    assert np.array_equal(host(src), es)
    assert np.array_equal(host(wstart), ew) and np.array_equal(host(key), ek)
    # the executor's pipeline on top of the expansion
    col = lambda i: [(L.OP_COL, i, 0, 0.0, 0)]
    (wstart, key, src), m = ops.scan_filter_project([wstart, key, src], [(L.OP_CMP_COL_IMM, 2, L.CMP_GE, 0.0, 0)], [col(0), col(1), col(2)],
                                                    stable=True)
    ge, gg = ops.gather([dev(ve), dev(vg)], src)
    ha = ops.HashAggState([torch.int32, torch.int64], [L.AGG_SUM, L.AGG_MIN, L.AGG_MAX, L.AGG_SUM, L.AGG_MIN],
                          max(1 << 12, 2 * m), ge.device)
    ha.update([key, wstart], [ge, ge, ge, gg, gg])
    (ok, ow), ov, oc = ha.finalize()
    ok, ow, oc = host(ok), host(ow), host(oc)
    ov = [host(v) for v in ov]
    o = np.lexsort((ow, ok))
    ro, rkey, rstart, lo, hi = R.hopping_window_ranges(ts, bs, size, hop)
    assert np.array_equal(ok[o], rkey) and np.array_equal(ow[o], rstart)
    assert np.array_equal(oc[o], hi - lo)
    assert np.array_equal(bits(ov[0][o]), bits(R.range_aggregate("sum", ve, lo, hi)))
    assert np.array_equal(ov[1][o], R.range_aggregate("min", ve, lo, hi))
    assert np.array_equal(ov[2][o], R.range_aggregate("max", ve, lo, hi))
    check_sum(ov[3][o], vg, lo, hi, "hop general sum")
    assert np.array_equal(ov[4][o], R.range_aggregate("min", vg, lo, hi))


# ------------------------------------------------------------------ session ids
@pytest.mark.parametrize("n", [2047, 2048, 2049, 2048 * 1024 - 1, 2048 * 1024, 2048 * 1024 + 1, 5_000_003])
def test_window_session_ids(qb, n):
    """ids = inclusive prefix sum of the new-session flags.  The scan works in tiles of 2048 rows and its block-sum pass
    carries between groups of 1024 tiles, so the sizes straddle 1 and 1024 tiles.  Timeout 0 keeps equal times in one session;
    a huge timeout leaves one session per key; the times are negative."""
    rng = np.random.default_rng(n)
    nkeys = 7
    time = np.sort(rng.integers(-n, 0, n)).astype(np.int64)           # about one tie per row
    by = draw_keys(rng, n, nkeys)
    order, seg = segmented(time, by, nkeys)
    ts, bs = time[order], by[order]
    dts, dbs = dev(ts), dev(bs)
    for timeout in (0, 3, 2 ** 62):
        flag = np.ones(n, dtype=np.int64)
        flag[1:] = (bs[1:] != bs[:-1]) | ((ts[1:] - ts[:-1]) > timeout)
        got = host(qb.ops.window_session_ids(dts, dbs, timeout))
        assert np.array_equal(got, np.cumsum(flag)), timeout
    assert got[-1] == len(np.unique(bs))


# ------------------------------------------------------------------ windows through the API at scale
_AGGD = {"avg_bid": "AVG(bid)", "max_ask": "MAX(ask)", "min_bid": "MIN(bid)", "sum_ask": "SUM(ask)", "n": "count(*)"}


def _check_api(res, kind, time, sym, bid, ask, ref, tcol="time"):
    """res (a pyarrow table of windowed_transform) against the reference ranges `ref` of the same rows."""
    import pyarrow as pa
    cols = {c: res[c] for c in res.column_names}
    t = cols[tcol]
    if pa.types.is_timestamp(t.type):
        t = t.cast(pa.int64())
    t = np.asarray(t.to_numpy(), dtype=np.int64)
    s = np.asarray(cols["symbol"].to_numpy(), dtype=np.int64)
    vals = {"bid": bid.astype(np.float64), "ask": ask.astype(np.float64)}
    if kind == "sliding":
        order, lo, hi = ref
        o = np.arange(len(t))
        assert np.array_equal(t, time[order]) and np.array_equal(s, sym[order])
    else:
        order, rkey, rstart, lo, hi = ref
        o = np.lexsort((t, s))
        assert np.array_equal(s[o], rkey) and np.array_equal(t[o], rstart)
    for name, (op, c) in {"avg_bid": ("avg", "bid"), "max_ask": ("max", "ask"), "min_bid": ("min", "bid"), "sum_ask": ("sum", "ask"),
                          "n": ("count", None)}.items():
        got = np.asarray(cols[name].to_numpy(), dtype=np.float64)[o]
        v = vals[c][order] if c else None
        check_agg(op, got, v, False, lo, hi, (kind, name))


@pytest.fixture(scope="module")
def tick_quotes(qb):
    from oracle import tpch_gen as G
    q = qb.synth.ticks(G.T_QUOTES, 2_000_000, 8000, columns=["time", "symbol", "bid", "ask"])
    return {k: host(v) for k, v in q.items()}


def test_windowed_transform_at_scale(qb, tick_quotes):
    """All four window types over 2 M quotes of 8 000 symbols (float32 bid / ask), once with int64 times cut into many small
    batches, once with a timestamp[ns] column and datetime.timedelta lengths (Window.ticks converts them to the column's unit)."""
    import pyarrow as pa
    from quokka_b200.df import QuokkaContext
    from quokka_b200.windowtypes import (HoppingWindow, OnCompletionTrigger, OnEventTrigger, SessionWindow, SlidingWindow,
                                         TumblingWindow)
    q = tick_quotes
    time, sym, bid, ask = q["time"], q["symbol"].astype(np.int64), q["bid"], q["ask"]
    slide, size, hop, tum, gap = 2_000_000, 2_500_000, 1_000_000, 1_000_000, 500_000
    refs = {"sliding": R.sliding_window_ranges(time, sym, slide), "hopping": R.hopping_window_ranges(time, sym, size, hop),
            "tumbling": R.hopping_window_ranges(time, sym, tum, tum), "session": R.session_window_ranges(time, sym, gap)}
    qc = QuokkaContext()
    ns = lambda x: datetime.timedelta(microseconds=x // 1000)
    for stamp, chunk in ((False, 65_536), (True, 1 << 26)):
        tarr = pa.array(time, type=pa.timestamp("ns")) if stamp else pa.array(time)
        table = pa.table({"time": tarr, "symbol": sym, "bid": bid, "ask": ask})
        L = ns if stamp else (lambda x: x)
        windows = {"sliding": (SlidingWindow("time", "symbol", L(slide), _AGGD), OnEventTrigger()),
                   "hopping": (HoppingWindow("time", "symbol", L(hop), L(size), _AGGD), OnCompletionTrigger()),
                   "tumbling": (TumblingWindow("time", "symbol", L(tum), _AGGD), OnCompletionTrigger()),
                   "session": (SessionWindow("time", "symbol", L(gap), _AGGD), OnCompletionTrigger())}
        qc.set_config("chunk_rows", chunk)
        try:
            for kind, (w, trig) in windows.items():
                res = qc.from_arrow_sorted(table, "time").windowed_transform(w, trig).collect()
                _check_api(res, "sliding" if kind == "sliding" else "grouped", time, sym, bid, ask, refs[kind])
        finally:
            qc.set_config("chunk_rows", 1 << 26)


# ------------------------------------------------------------------ more keys than the shared-memory tables hold
@pytest.mark.parametrize("nparts", [16_383, 16_384, 16_385, 40_961, 100_000, 1 << 20])
@pytest.mark.parametrize("dtype", [np.int32, np.int64])
def test_partition_code_any_nparts(qb, nparts, dtype):
    """CODE partition = stable argsort of the clamped codes, part_offsets from their counts.  16 384 parts is the largest
    table that fits shared memory; above it the partition runs one stable pass per 14-bit digit."""
    n = 1_000_003
    rng = np.random.default_rng(nparts)
    code = (rng.random(n) ** 2 * nparts).astype(np.int64)           # skewed: large and empty partitions
    code[::97] = -5                                                  # out of range: clamped to 0 ...
    code[13::101] = nparts + (1 << 33 if dtype == np.int64 else 3)   # ... and to nparts - 1
    code[-1] = nparts - 1
    code = code.astype(dtype)
    clamped = np.clip(code.astype(np.int64), 0, nparts - 1)
    dest, offs = qb.ops.partition_plan(dev(code), nparts, qb.L.PART_CODE)
    out = host(qb.ops.scatter([dev(np.arange(n, dtype=np.int32))], dest)[0])
    assert np.array_equal(out, np.argsort(clamped, kind="stable"))
    assert np.array_equal(host(offs), np.concatenate([[0], np.cumsum(np.bincount(clamped, minlength=nparts))]))


def test_partition_mod_keeps_its_limit(qb):
    key = dev(np.arange(1000, dtype=np.int64))
    qb.ops.partition_plan(key, 16_384)
    with pytest.raises(qb.L.QkError, match="nparts"):
        qb.ops.partition_plan(key, 16_385)


def _asof_inputs(rng, nt, nq, n_by):
    lt = np.sort(rng.integers(0, 10 ** 8, nt)).astype(np.int64)
    rt = np.sort(rng.integers(0, 10 ** 8, nq)).astype(np.int64)
    lb = rng.integers(0, n_by, nt).astype(np.int32)
    rb = rng.integers(0, n_by, nq).astype(np.int32)
    lb[-1] = rb[-1] = n_by - 1
    return lt, lb, rt, rb


def test_asof_merge_table_limit(qb):
    """The merge kernel's table holds 40 960 keys (160 KB of int32); one more and it declines."""
    rng = np.random.default_rng(40_960)
    lt, lb, rt, rb = _asof_inputs(rng, 100_000, 400_000, 40_960)
    out, _ = qb.ops.asof_merge(dev(lt), dev(lb), dev(rt), dev(rb), 40_960)
    assert np.array_equal(host(out), R.asof_backward_fast(lt, lb, rt, rb))
    assert qb.ops.asof_merge(dev(lt), dev(lb), dev(rt), dev(rb), 40_961) == (None, None)


@pytest.mark.parametrize("n_by", [16_385, 40_961, 100_000])
def test_asof_backward_many_keys(qb, n_by):
    rng = np.random.default_rng(n_by)
    lt, lb, rt, rb = _asof_inputs(rng, 200_000, 500_000, n_by)
    got = host(qb.ops.asof_backward(dev(lt), dev(lb), dev(rt), dev(rb), n_by))
    exp = R.asof_backward_fast(lt, lb, rt, rb)
    assert (exp >= 0).sum() > 100_000
    assert np.array_equal(got, exp)


@pytest.mark.parametrize("strings", [True, False])
def test_join_asof_many_symbols(qb, monkeypatch, strings):
    """join_asof with 50 000 string symbols, and with integer symbol ids up to 100 000: too many keys for the merge kernel,
    so the executor keeps the whole quote state and searches it (ops.asof_backward)."""
    import pyarrow as pa
    from quokka_b200 import executors as X
    from quokka_b200.df import QuokkaContext
    rng = np.random.default_rng(50_000 + strings)
    nsym = 50_000 if strings else 100_000
    lt, lb, rt, rb = _asof_inputs(rng, 100_000, 500_000, nsym)
    if strings:
        names = np.array([f"S{i:05d}" for i in range(nsym)], dtype=object)
        tsym, qsym = pa.array(list(names[lb])), pa.array(list(names[rb]))
    else:
        tsym, qsym = pa.array(lb.astype(np.int64)), pa.array(rb.astype(np.int64))
    trades = pa.table({"time": lt, "symbol": tsym, "it": np.arange(len(lt), dtype=np.int64)})
    quotes = pa.table({"time": rt, "symbol": qsym, "iq": np.arange(len(rt), dtype=np.int64)})
    searched = []
    real = X.ops.asof_backward
    monkeypatch.setattr(X.ops, "asof_backward", lambda *a: searched.append(a[-1]) or real(*a))
    qc = QuokkaContext()
    res = qc.from_arrow_sorted(trades, "time").join_asof(qc.from_arrow_sorted(quotes, "time"), on="time", by="symbol").collect()
    assert searched and min(searched) > 40_960
    it = res["it"].to_numpy()
    iq = res["iq"].fill_null(-1).to_numpy()[np.argsort(it)]
    assert np.array_equal(np.sort(it), np.arange(len(lt)))
    assert np.array_equal(iq, R.asof_backward_fast(lt, lb, rt, rb))


def test_windowed_transform_many_keys(qb):
    """20 000 keys: the window executors segment their rows with a CODE partition of more than 16 384 parts."""
    import pyarrow as pa
    from quokka_b200.df import QuokkaContext
    from quokka_b200.windowtypes import OnCompletionTrigger, OnEventTrigger, SlidingWindow, TumblingWindow
    rng = np.random.default_rng(20_000)
    n, nkeys = 300_000, 20_000
    time = np.sort(rng.integers(0, 10 ** 7, n)).astype(np.int64)
    sym = rng.integers(0, nkeys, n).astype(np.int64)
    sym[-1] = nkeys - 1
    bid = (rng.integers(0, 100_000, n) / 100).astype(np.float32)
    ask = (rng.integers(0, 100_000, n) / 100).astype(np.float32)
    table = pa.table({"time": time, "symbol": sym, "bid": bid, "ask": ask})
    qc = QuokkaContext()
    res = qc.from_arrow_sorted(table, "time").windowed_transform(SlidingWindow("time", "symbol", 200_000, _AGGD), OnEventTrigger()).collect()
    _check_api(res, "sliding", time, sym, bid, ask, R.sliding_window_ranges(time, sym, 200_000))
    res = qc.from_arrow_sorted(table, "time").windowed_transform(TumblingWindow("time", "symbol", 100_000, _AGGD), OnCompletionTrigger()).collect()
    _check_api(res, "grouped", time, sym, bid, ask, R.hopping_window_ranges(time, sym, 100_000, 100_000))
