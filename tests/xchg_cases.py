"""Exchange-level parity checks of runtime.Exchange, run by the multi-GPU check (tests/dist_xchg_check.py, over the
peer-memory link or NCCL) and on gloo ranks (tests/test_dist_gloo_exchange.py).  Every rank draws the SAME global table
from a seed, keeps its shard, runs the exchange and checks what it received against numpy: rows with key % world == rank,
per source rank in source order (the partition is stable), bit-exact.  Covers hash-partitioned edges at several sizes,
ranks with nothing to send, a hash edge with a validity mask, broadcast with a validity mask and per-rank dictionaries, single owner, and the small
all-gather."""
import numpy as np
import torch
import torch.distributed as dist


def _table_of(dev, cols, lo, hi, dicts=None, valid=None):
    from quokka_b200.columns import DeviceColumn, DeviceTable
    out = {}
    for n, v in cols.items():
        out[n] = DeviceColumn(torch.from_numpy(np.ascontiguousarray(v[lo:hi])).to(dev), (dicts or {}).get(n), None,
                              None if valid is None or n not in valid else torch.from_numpy(np.ascontiguousarray(valid[n][lo:hi])).to(dev))
    return DeviceTable(out)


def _shard(n, r):
    w = dist.get_world_size()
    return n * r // w, n * (r + 1) // w


def check_hash(ex, dev, n, seed, empty_ranks=(), tag="", masked=False):
    """masked: column "a" carries a validity mask, which must reach the receivers with its rows."""
    from quokka_b200.edge import apply_partitioner
    from quokka_b200.target_info import HashPartitioner
    w, me = dist.get_world_size(), dist.get_rank()
    rng = np.random.default_rng(seed)
    cols = {"k": rng.integers(0, 1 << 40, n), "a": rng.random(n), "b": rng.integers(-100, 100, n).astype(np.int32),
            "c": rng.integers(0, 200, n).astype(np.uint8)}
    valid = {"a": (rng.random(n) < 0.6).astype(np.uint8)} if masked else None
    lo, hi = _shard(n, me)
    if me in empty_ranks:
        hi = lo
    t = _table_of(dev, cols, lo, hi, valid=valid)
    parts = apply_partitioner(HashPartitioner("k"), t, me, w) if hi > lo else {}
    got = ex(parts, w, edge_key=("hash", tag))
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
    w, me = dist.get_world_size(), dist.get_rank()
    rng = np.random.default_rng(20)
    n = 10_007
    words = [f"w{i}" for i in range(50)]
    mydict = [words[(i * 7 + me * 3) % 50] for i in range(50)]                   # a different code assignment on every rank
    codes = rng.integers(0, 50, n)
    lo, hi = _shard(n, me)
    cols = {"x": rng.random(n), "s": codes.astype(np.int32)}
    valid = {"x": (rng.random(n) < 0.7).astype(np.uint8)}
    t = _table_of(dev, cols, lo, hi, {"s": mydict}, valid)
    got = ex({r: t for r in range(w)}, w, edge_key=("bcast",))
    assert sorted(set(g.src_rank for g in got)) == list(range(w))
    for s in range(w):
        a, b = _shard(n, s)
        mine_ = [g for g in got if g.src_rank == s]
        assert np.array_equal(np.concatenate([g["x"].data.cpu().numpy() for g in mine_]), cols["x"][a:b])
        assert np.array_equal(np.concatenate([g["x"].valid.cpu().numpy() for g in mine_]), valid["x"][a:b])
        sdict = [words[(i * 7 + s * 3) % 50] for i in range(50)]
        assert [g["s"].dictionary[c] for g in mine_ for c in g["s"].data.cpu().numpy()] == [sdict[c] for c in cols["s"][a:b]], "values survive the re-coding"
    got = ex({0: t}, 1, single_owner=0, edge_key=("single",))
    assert (sorted(set(g.src_rank for g in got)) == list(range(w))) if me == 0 else (got == [])
    if me == 0:
        assert np.array_equal(np.concatenate([g["x"].data.cpu().numpy() for g in got]), cols["x"])


def run_all(ex, dev):
    w, me = dist.get_world_size(), dist.get_rank()
    for n, seed in ((0, 1), (1, 2), (5, 3), (2047, 4), (2049, 5), (100_003, 6), (3_000_017, 7)):
        check_hash(ex, dev, n, seed, tag=f"hash{n}")
    check_hash(ex, dev, 50_000, 8, empty_ranks=(0,), tag="empty0")
    check_hash(ex, dev, 50_000, 9, empty_ranks=tuple(range(1, w)), tag="only0")
    check_hash(ex, dev, 100_003, 10, tag="masked", masked=True)
    check_broadcast_and_single_owner(ex, dev)
    rows = ex.allgather_words([me * 10 + 1, 7])
    assert rows == [[r * 10 + 1, 7] for r in range(w)]
