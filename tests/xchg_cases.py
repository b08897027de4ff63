"""Exchange-level parity checks of runtime.Exchange, run by the multi-GPU check (tests/dist_xchg_check.py, over the
peer-memory link or NCCL), on gloo ranks (tests/test_dist_gloo_exchange.py) and on the in-process link (tests/inproc_link.py:
tests/test_gpu_xchg.py on one GPU, tests/test_xchg_cpu.py over the numpy shim).  Every rank draws the SAME global table
from a seed, keeps its shard, runs the exchange and checks what it received against numpy: rows with key % world == rank,
per source rank in source order (the partition is stable), bit-exact, in a list whose source ranks never decrease (also when
the payload went in rounds); and the bytes it sent to other ranks (validity masks
included) and every rank's received-row total on the edge, exactly.  Covers hash-partitioned edges at several sizes,
ranks with nothing to send, validity masks, edges of 20 columns and of 12 masked columns (24 buffers), broadcast with a
validity mask and per-rank dictionaries, vector columns, a hash edge whose dictionaries differ per rank and grow, single
owner, and the small all-gather.  `run_rounds` is for a link with a small mailbox: payloads that go in rounds, one of them
skewed so that a round still overflows a receiver.  World and rank come from runtime.world_size() / rank()."""
import numpy as np
import torch

from quokka_b200 import runtime


def _table_of(dev, cols, lo, hi, dicts=None, valid=None):
    from quokka_b200.columns import DeviceColumn, DeviceTable
    out = {}
    for n, v in cols.items():
        out[n] = DeviceColumn(torch.from_numpy(np.ascontiguousarray(v[lo:hi])).to(dev), (dicts or {}).get(n), None,
                              None if valid is None or n not in valid else torch.from_numpy(np.ascontiguousarray(valid[n][lo:hi])).to(dev))
    return DeviceTable(out)


def _shard(n, r):
    w = runtime.world_size()
    return n * r // w, n * (r + 1) // w


def _width(v: np.ndarray) -> int:
    """Bytes of one row of a column."""
    return v.dtype.itemsize * (v.shape[1] if v.ndim == 2 else 1)


def _check_source_order(got, what):
    """The received tables come per source rank in rank order, a source's rounds one after the other: consumers fed through
    the task graph see them in list order."""
    srcs = [g.src_rank for g in got]
    assert srcs == sorted(srcs), (what, runtime.rank(), srcs)


def _check_accounting(ex, edge_key, sent_before, sent, recv_rows):
    """ex.bytes_sent grew by exactly `sent` bytes and every rank knows the rows each rank has received on the edge."""
    assert ex.bytes_sent - sent_before == sent, (edge_key, runtime.rank(), ex.bytes_sent - sent_before, sent)
    assert ex.recv_totals[edge_key] == [int(x) for x in recv_rows], (edge_key, ex.recv_totals[edge_key], list(recv_rows))


def _skewed_keys(rng, n, w):
    """Keys of which 30 % go to rank 0 and the rest evenly to the others, every shard sorted by key: a shard's rows for one
    rank are one contiguous run, so a round (a slice of every shard) concentrates them and can overflow that receiver."""
    g = np.where(rng.random(n) < 0.3, 0, rng.integers(1, max(2, w), n) % w)
    k = g + w * rng.integers(0, 1 << 30, n)
    for s in range(w):
        a, b = _shard(n, s)
        k[a:b] = k[a:b][np.argsort(k[a:b] % w * (1 << 40) + k[a:b] // w, kind="stable")]
    return k


def check_hash(ex, dev, n, seed, empty_ranks=(), tag="", masked=False, skew=False):
    """masked: column "a" carries a validity mask, which must reach the receivers with its rows.  skew: see _skewed_keys."""
    from quokka_b200.edge import apply_partitioner
    from quokka_b200.target_info import HashPartitioner
    w, me = runtime.world_size(), runtime.rank()
    rng = np.random.default_rng(seed)
    cols = {"k": _skewed_keys(rng, n, w) if skew else rng.integers(0, 1 << 40, n), "a": rng.random(n),
            "b": rng.integers(-100, 100, n).astype(np.int32), "c": rng.integers(0, 200, n).astype(np.uint8)}
    valid = {"a": (rng.random(n) < 0.6).astype(np.uint8)} if masked else None
    lo, hi = _shard(n, me)
    if me in empty_ranks:
        hi = lo
    t = _table_of(dev, cols, lo, hi, valid=valid)
    parts = apply_partitioner(HashPartitioner("k"), t, me, w) if hi > lo else {}
    sent0 = ex.bytes_sent
    got = ex(parts, w, edge_key=("hash", tag))
    _check_source_order(got, tag)
    nonempty = [np.arange(*_shard(n, s)) for s in range(w) if s not in empty_ranks]
    dest_all = np.concatenate(nonempty) if nonempty else np.zeros(0, np.int64)
    recv_rows = np.bincount(cols["k"][dest_all] % w, minlength=w)
    row_bytes = sum(_width(v) for v in cols.values()) + (1 if masked else 0)
    _check_accounting(ex, ("hash", tag), sent0, int((cols["k"][lo:hi] % w != me).sum()) * row_bytes, recv_rows)
    exp = []
    for s in range(w):
        a, b = _shard(n, s)
        if s in empty_ranks:
            b = a
        sel = np.nonzero(cols["k"][a:b] % w == me)[0] + a
        if len(sel):
            exp.append(sel)
    # one table per source rank, or several per source when the payload went in rounds: rows per source, in order
    srcs = sorted(set(g.src_rank for g in got))
    assert len(srcs) == len(exp), (tag, me, len(got), len(exp))
    for s_, sel in zip(srcs, exp):
        for name, v in cols.items():
            have = np.concatenate([g[name].data.cpu().numpy() for g in got if g.src_rank == s_])
            assert np.array_equal(have, v[sel]), (tag, me, name)
        if masked:
            have = np.concatenate([g["a"].valid.cpu().numpy() for g in got if g.src_rank == s_])
            assert np.array_equal(have, valid["a"][sel]), (tag, me, "valid")


def check_broadcast_and_single_owner(ex, dev):
    """Broadcast and single owner, with a validity mask on one column and a different dictionary on every rank."""
    w, me = runtime.world_size(), runtime.rank()
    rng = np.random.default_rng(20)
    n = 10_007
    words = [f"w{i}" for i in range(50)]
    mydict = [words[(i * 7 + me * 3) % 50] for i in range(50)]                   # a different code assignment on every rank
    codes = rng.integers(0, 50, n)
    lo, hi = _shard(n, me)
    cols = {"x": rng.random(n), "s": codes.astype(np.int32)}
    valid = {"x": (rng.random(n) < 0.7).astype(np.uint8)}
    t = _table_of(dev, cols, lo, hi, {"s": mydict}, valid)
    sent0, row_bytes = ex.bytes_sent, 8 + 4 + 1
    got = ex({r: t for r in range(w)}, w, edge_key=("bcast",))
    _check_source_order(got, "bcast")
    _check_accounting(ex, ("bcast",), sent0, (hi - lo) * (w - 1) * row_bytes, [n] * w)
    assert sorted(set(g.src_rank for g in got)) == list(range(w))
    for s in range(w):
        a, b = _shard(n, s)
        mine_ = [g for g in got if g.src_rank == s]
        assert np.array_equal(np.concatenate([g["x"].data.cpu().numpy() for g in mine_]), cols["x"][a:b])
        assert np.array_equal(np.concatenate([g["x"].valid.cpu().numpy() for g in mine_]), valid["x"][a:b])
        sdict = [words[(i * 7 + s * 3) % 50] for i in range(50)]
        assert [g["s"].dictionary[c] for g in mine_ for c in g["s"].data.cpu().numpy()] == [sdict[c] for c in cols["s"][a:b]], "values survive the re-coding"
    sent0 = ex.bytes_sent
    got = ex({0: t}, 1, single_owner=0, edge_key=("single",))
    _check_source_order(got, "single")
    _check_accounting(ex, ("single",), sent0, 0 if me == 0 else (hi - lo) * row_bytes, [n] + [0] * (w - 1))
    assert (sorted(set(g.src_rank for g in got)) == list(range(w))) if me == 0 else (got == [])
    if me == 0:
        # per source rank in rank order (when the payload went in rounds, every round brings a table from each source)
        assert np.array_equal(np.concatenate([g["x"].data.cpu().numpy() for s in range(w) for g in got if g.src_rank == s]), cols["x"])


_WIDE_DTYPES = (np.int64, np.float64, np.int32, np.uint8, np.float32)


def check_wide(ex, dev, kind, ncols, masked=False, n=30_011, seed=30):
    """A hash (`kind` = "hash") or broadcast ("bcast") edge of `ncols` columns of every scalar dtype, each with a validity
    mask when `masked`: more buffers than one kernel call of the other operators takes (QK_MAX_COLS)."""
    from quokka_b200.edge import apply_partitioner
    from quokka_b200.target_info import HashPartitioner
    w, me = runtime.world_size(), runtime.rank()
    rng = np.random.default_rng(seed + ncols + (100 if masked else 0))
    cols = {"k": rng.integers(-(1 << 40), 1 << 40, n)}
    for i in range(1, ncols):
        dt = _WIDE_DTYPES[i % len(_WIDE_DTYPES)]
        cols[f"c{i:02d}"] = (rng.random(n) * 1e6 - 5e5).astype(dt) if dt in (np.float32, np.float64) else \
            rng.integers(np.iinfo(dt).min, np.iinfo(dt).max, n, dtype=dt, endpoint=True)
    valid = {name: (rng.random(n) < 0.5 + 0.02 * i).astype(np.uint8) for i, name in enumerate(cols)} if masked else None
    lo, hi = _shard(n, me)
    t = _table_of(dev, cols, lo, hi, valid=valid)
    key = (kind, ncols, masked)
    row_bytes = sum(_width(v) for v in cols.values()) + (len(cols) if masked else 0)
    sent0 = ex.bytes_sent
    if kind == "hash":
        got = ex(apply_partitioner(HashPartitioner("k"), t, me, w), w, edge_key=key)
        mine_ = [np.nonzero(cols["k"][slice(*_shard(n, s))] % w == me)[0] + _shard(n, s)[0] for s in range(w)]
        _check_accounting(ex, key, sent0, int((cols["k"][lo:hi] % w != me).sum()) * row_bytes, np.bincount(cols["k"] % w, minlength=w))
    else:
        got = ex({r: t for r in range(w)}, w, edge_key=key)
        mine_ = [np.arange(*_shard(n, s)) for s in range(w)]
        _check_accounting(ex, key, sent0, (hi - lo) * (w - 1) * row_bytes, [n] * w)
    _check_source_order(got, key)
    mine_ = [(s, sel) for s, sel in enumerate(mine_) if len(sel)]
    assert sorted(set(g.src_rank for g in got)) == [s for s, _ in mine_], (key, me)
    for s, sel in mine_:
        part = [g for g in got if g.src_rank == s]
        for name, v in cols.items():
            assert np.array_equal(np.concatenate([g[name].data.cpu().numpy() for g in part]), v[sel]), (key, me, s, name)
            if masked:
                assert np.array_equal(np.concatenate([g[name].valid.cpu().numpy() for g in part]), valid[name][sel]), (key, me, s, name)


def check_vectors(ex, dev, n=4_099, seed=40):
    """A broadcast of f32 and f16 vector columns (whole rows of 7 x 4 and 5 x 2 bytes) next to a scalar column."""
    w, me = runtime.world_size(), runtime.rank()
    rng = np.random.default_rng(seed)
    cols = {"id": np.arange(n, dtype=np.int64) * 3 - 7, "v32": rng.standard_normal((n, 7)).astype(np.float32),
            "v16": rng.standard_normal((n, 5)).astype(np.float16)}
    lo, hi = _shard(n, me)
    t = _table_of(dev, cols, lo, hi)
    sent0 = ex.bytes_sent
    got = ex({r: t for r in range(w)}, w, edge_key=("vectors",))
    _check_source_order(got, "vectors")
    _check_accounting(ex, ("vectors",), sent0, (hi - lo) * (w - 1) * (8 + 28 + 10), [n] * w)
    srcs = [s for s in range(w) if _shard(n, s)[1] > _shard(n, s)[0]]
    assert sorted(set(g.src_rank for g in got)) == srcs
    for s in srcs:
        a, b = _shard(n, s)
        for name, v in cols.items():
            have = np.concatenate([g[name].data.cpu().numpy() for g in got if g.src_rank == s])
            assert have.dtype == v.dtype and np.array_equal(have.view(np.uint8), v[a:b].view(np.uint8)), (me, s, name)


def check_dictionaries(ex, dev, n=20_003, seed=50):
    """A hash edge whose dictionary column has a different code assignment and a different subset of the values on every
    rank, used twice: the second time one rank's dictionary has grown, so the schemas are negotiated again (on the link:
    _share_objects), and rank 0 has no rows to send but receives.  Values must survive the re-coding."""
    from quokka_b200.edge import apply_partitioner
    from quokka_b200.target_info import HashPartitioner
    w, me = runtime.world_size(), runtime.rank()
    words = [f"v{i:03d}" for i in range(120)]

    def dict_of(r, grown):
        sub = [words[(i * 11 + r * 5) % 120] for i in range(60 + 7 * r)]
        return sub + ([f"new{r}-{i}" for i in range(9)] if grown and r == w - 1 else [])

    for call, grown in enumerate((False, True)):
        rng = np.random.default_rng(seed + call)
        k = rng.integers(0, 1 << 40, n)
        sizes = [len(dict_of(r, grown)) for r in range(w)]
        lo, hi = _shard(n, me)
        codes = np.zeros(n, dtype=np.int32)
        for r in range(w):
            a, b = _shard(n, r)
            codes[a:b] = rng.integers(0, sizes[r], b - a)
        empty = (0,) if grown else ()
        if me in empty:
            hi = lo
        t = _table_of(dev, {"k": k, "s": codes}, lo, hi, {"s": dict_of(me, grown)})
        parts = apply_partitioner(HashPartitioner("k"), t, me, w) if hi > lo else {}
        got = ex(parts, w, edge_key=("dicts",))
        _check_source_order(got, ("dicts", call))
        for s in range(w):
            if s in empty:
                continue
            a, b = _shard(n, s)
            sel = np.nonzero(k[a:b] % w == me)[0] + a
            part = [g for g in got if g.src_rank == s]
            assert len(part) == (1 if len(sel) else 0), (me, s, call)
            if len(sel):
                sd = dict_of(s, grown)
                assert np.array_equal(part[0]["k"].data.cpu().numpy(), k[sel])
                assert [part[0]["s"].dictionary[c] for c in part[0]["s"].data.cpu().numpy()] == [sd[c] for c in codes[sel]], (me, s, call)


def run_all(ex, dev):
    w, me = runtime.world_size(), runtime.rank()
    for n, seed in ((0, 1), (1, 2), (5, 3), (2047, 4), (2049, 5), (100_003, 6), (3_000_017, 7)):
        check_hash(ex, dev, n, seed, tag=f"hash{n}")
    check_hash(ex, dev, 50_000, 8, empty_ranks=(0,), tag="empty0")
    check_hash(ex, dev, 50_000, 9, empty_ranks=tuple(range(1, w)), tag="only0")
    check_hash(ex, dev, 100_003, 10, tag="masked", masked=True)
    check_broadcast_and_single_owner(ex, dev)
    check_wide(ex, dev, "hash", 20)
    check_wide(ex, dev, "bcast", 20)
    check_wide(ex, dev, "hash", 12, masked=True)
    check_wide(ex, dev, "bcast", 12, masked=True)
    check_vectors(ex, dev)
    check_dictionaries(ex, dev)
    rows = ex.allgather_words([me * 10 + 1, 7])
    assert rows == [[r * 10 + 1, 7] for r in range(w)]


def run_rounds(ex, dev):
    """For a link whose mailbox is far smaller than the payloads (~64 KB): a hash edge, a broadcast and a single owner go
    in rounds; the skewed hash edge overflows a receiver inside a round, so the rounds split again."""
    check_hash(ex, dev, 60_001, 11, tag="rounds")
    check_broadcast_and_single_owner(ex, dev)
    check_hash(ex, dev, 60_001, 12, tag="skewed", skew=True)
    check_wide(ex, dev, "hash", 12, masked=True, n=9_001)
