"""Every caller-provided workspace has one layout per kernel (csrc/common.cuh Carve): the same function sizes it for
qk_*_workspace_bytes and hands out its pieces in the entry point, which checks the caller's buffer against that total.

Without a GPU: every sizing function over a grid of shapes (empty and one-row inputs, each kernel's tile boundaries, 2^31 - 1
rows, nparts on both sides of the radix partition's 16 384, n_by on both sides of the as-of merge's 160 KB table, Gram k of
1 / 8 / 1031, knn q and k at their bounds, invalid arguments) returns the pinned byte counts below.  The sizes depend on the
SM count, so the queries run in a process that sees no device, where sm_count() takes its no-device value of 132 (the H100
SXM); the table then holds on any machine.  The Parquet entries are min(pages, 8 x 132) slots, rounded up to whole
4-warp CTAs, times the slot size.

On the GPU: a workspace one byte short of its size is refused with QK_ERR_CAPACITY before any kernel runs, except where a
short workspace has a defined fallback (the unordered scan runs the interpreter, Parquet inflate keeps fewer pages in
flight) or none is needed (a shift without a key)."""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from quokka_b200 import _lib as L

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

PINNED = {
    "qk_sort_workspace_bytes": [
        ((-1,), 0), ((0,), 3175680), ((1,), 3176704), ((4095,), 3273984), ((4096,), 3273984), ((4097,), 3275008),
        ((1000003,), 27176704), ((2147483647,), 51542783232),
    ],
    "qk_topk_workspace_bytes": [
        ((-1,), 0), ((0,), 1280), ((1,), 1536), ((4095,), 34048), ((4096,), 34048), ((4097,), 34304), ((1000003,), 8001536),
        ((2147483647,), 17179870464),
    ],
    "qk_window_session_workspace_bytes": [
        ((-1,), 0), ((0,), 256), ((1,), 512), ((2047,), 8448), ((2048,), 8448), ((2049,), 8704), ((1000003,), 4004352),
        ((2147483647,), 8598323456),
    ],
    "qk_shift_workspace_bytes": [
        ((-1,), 0), ((0,), 256), ((1,), 512), ((2047,), 8448), ((2048,), 8448), ((2049,), 8704), ((1000003,), 4000512),
        ((2147483647,), 8589934848),
    ],
    "qk_scan_workspace_bytes": [
        ((0,), 16704), ((1,), 16704), ((31,), 16704), ((32,), 16704), ((33,), 16704), ((2047,), 16960), ((2048,), 16960),
        ((2049,), 16960), ((1000003,), 141632), ((2147483647,), 268452160), ((6000000000,), 750016576),
    ],
    "qk_scan_agg_workspace_bytes": [
        ((0, 1), 0), ((-1, 1), 0), ((1, -1), 0), ((1, 0), 16384), ((1, 1), 16384), ((6, 5), 294912), ((4096, 0), 67108864),
        ((4096, 8), 301989888),
    ],
    "qk_hashagg_state_bytes": [
        ((0, 1, 1), 0), ((-1024, 1, 1), 0), ((1, 1, 0), 1280), ((1024, 1, 0), 36864), ((1024, 2, 5), 69632),
        ((2097152, 3, 8), 192937984), ((134217728, 1, 1), 4831838208),
    ],
    "qk_partition_workspace_bytes": [
        ((-1, -1), 0), ((-1, 0), 0), ((-1, 1), 0), ((-1, 2), 0), ((-1, 8), 0), ((-1, 16383), 0), ((-1, 16384), 0),
        ((-1, 16385), 0), ((-1, 1048576), 0), ((-1, 2147483647), 0), ((0, -1), 0), ((0, 0), 0), ((0, 1), 768),
        ((0, 2), 768), ((0, 8), 768), ((0, 16383), 327680), ((0, 16384), 327680), ((0, 16385), 459008),
        ((0, 1048576), 459008), ((0, 2147483647), 459008), ((1, -1), 0), ((1, 0), 0), ((1, 1), 768), ((1, 2), 768),
        ((1, 8), 768), ((1, 16383), 524288), ((1, 16384), 524288), ((1, 16385), 656640), ((1, 1048576), 656640),
        ((1, 2147483647), 656640), ((4095, -1), 0), ((4095, 0), 0), ((4095, 1), 768), ((4095, 2), 768), ((4095, 8), 768),
        ((4095, 16383), 524288), ((4095, 16384), 524288), ((4095, 16385), 721152), ((4095, 1048576), 721152),
        ((4095, 2147483647), 721152), ((4096, -1), 0), ((4096, 0), 0), ((4096, 1), 768), ((4096, 2), 768), ((4096, 8), 768),
        ((4096, 16383), 524288), ((4096, 16384), 524288), ((4096, 16385), 721152), ((4096, 1048576), 721152),
        ((4096, 2147483647), 721152), ((4097, -1), 0), ((4097, 0), 0), ((4097, 1), 768), ((4097, 2), 768), ((4097, 8), 768),
        ((4097, 16383), 720896), ((4097, 16384), 720896), ((4097, 16385), 918784), ((4097, 1048576), 918784),
        ((4097, 2147483647), 918784), ((1000003, -1), 0), ((1000003, 0), 0), ((1000003, 1), 3328), ((1000003, 2), 6400),
        ((1000003, 8), 24064), ((1000003, 16383), 48494080), ((1000003, 16384), 48496640), ((1000003, 16385), 64628992),
        ((1000003, 1048576), 64628992), ((1000003, 2147483647), 64628992), ((2147483647, -1), 0), ((2147483647, 0), 0),
        ((2147483647, 1), 99072), ((2147483647, 2), 197376), ((2147483647, 8), 787200), ((2147483647, 16383), 50656256),
        ((2147483647, 16384), 50659328), ((2147483647, 16385), 34410529024), ((2147483647, 1048576), 34410529024),
        ((2147483647, 2147483647), 34410529024),
    ],
    "qk_asof_workspace_bytes": [
        ((-1, -1), 0), ((-1, 0), 0), ((-1, 1), 0), ((-1, 8000), 0), ((-1, 16384), 0), ((-1, 16385), 0), ((-1, 1000000), 0),
        ((0, -1), 0), ((0, 0), 0), ((0, 1), 1024), ((0, 8000), 224256), ((0, 16384), 459008), ((0, 16385), 590336),
        ((0, 1000000), 8459264), ((1, -1), 0), ((1, 0), 0), ((1, 1), 1792), ((1, 8000), 321024), ((1, 16384), 656384),
        ((1, 16385), 788736), ((1, 1000000), 8657664), ((1000003, -1), 0), ((1000003, 0), 0), ((1000003, 1), 16004352),
        ((1000003, 8000), 39745024), ((1000003, 16384), 64628736), ((1000003, 16385), 80761088),
        ((1000003, 1000000), 88630016), ((2147483647, -1), 0), ((2147483647, 0), 0), ((2147483647, 1), 34359837696),
        ((2147483647, 8000), 34410266624), ((2147483647, 16384), 34410529024), ((2147483647, 16385), 68770398720),
        ((2147483647, 1000000), 68778267648),
    ],
    "qk_asof_merge_workspace_bytes": [
        ((0, 0, -1), 0), ((0, 0, 0), 0), ((0, 0, 1), 4608), ((0, 0, 8000), 16896256), ((0, 0, 40960), 21627136),
        ((0, 0, 40961), 0), ((1, 0, -1), 0), ((1, 0, 0), 0), ((1, 0, 1), 4608), ((1, 0, 8000), 16896256),
        ((1, 0, 40960), 21627136), ((1, 0, 40961), 0), ((0, 1, -1), 0), ((0, 1, 0), 0), ((0, 1, 1), 4608),
        ((0, 1, 8000), 16896256), ((0, 1, 40960), 21627136), ((0, 1, 40961), 0), ((-1, 5, -1), 0), ((-1, 5, 0), 0),
        ((-1, 5, 1), 0), ((-1, 5, 8000), 0), ((-1, 5, 40960), 0), ((-1, 5, 40961), 0), ((5, -1, -1), 0), ((5, -1, 0), 0),
        ((5, -1, 1), 0), ((5, -1, 8000), 0), ((5, -1, 40960), 0), ((5, -1, 40961), 0), ((1023, 0, -1), 0),
        ((1023, 0, 0), 0), ((1023, 0, 1), 4608), ((1023, 0, 8000), 16896256), ((1023, 0, 40960), 21627136),
        ((1023, 0, 40961), 0), ((1024, 0, -1), 0), ((1024, 0, 0), 0), ((1024, 0, 1), 4608), ((1024, 0, 8000), 16896256),
        ((1024, 0, 40960), 21627136), ((1024, 0, 40961), 0), ((1000, 25, -1), 0), ((1000, 25, 0), 0), ((1000, 25, 1), 4608),
        ((1000, 25, 8000), 16896256), ((1000, 25, 40960), 21627136), ((1000, 25, 40961), 0), ((1025, 0, -1), 0),
        ((1025, 0, 0), 0), ((1025, 0, 1), 4608), ((1025, 0, 8000), 16896256), ((1025, 0, 40960), 21627136),
        ((1025, 0, 40961), 0), ((1000000, 4000000, -1), 0), ((1000000, 4000000, 0), 0), ((1000000, 4000000, 1), 82688),
        ((1000000, 4000000, 8000), 16974336), ((1000000, 4000000, 40960), 21705216), ((1000000, 4000000, 40961), 0),
        ((2147483647, 2147483647, -1), 0), ((2147483647, 2147483647, 0), 0), ((2147483647, 2147483647, 1), 67113472),
        ((2147483647, 2147483647, 8000), 84005120), ((2147483647, 2147483647, 40960), 88736000),
        ((2147483647, 2147483647, 40961), 0),
    ],
    "qk_gram_workspace_bytes": [
        ((-1, -1), 0), ((-1, 0), 0), ((-1, 1), 0), ((-1, 7), 0), ((-1, 8), 0), ((-1, 9), 0), ((-1, 31), 0), ((-1, 32), 0),
        ((-1, 1031), 0), ((0, -1), 0), ((0, 0), 0), ((0, 1), 1024), ((0, 7), 1024), ((0, 8), 8704), ((0, 9), 8704),
        ((0, 31), 8960), ((0, 32), 33536), ((0, 1031), 5915392), ((1, -1), 0), ((1, 0), 0), ((1, 1), 1024), ((1, 7), 1024),
        ((1, 8), 8704), ((1, 9), 8704), ((1, 31), 8960), ((1, 32), 33536), ((1, 1031), 5915392), ((7, -1), 0), ((7, 0), 0),
        ((7, 1), 1024), ((7, 7), 1024), ((7, 8), 8704), ((7, 9), 8704), ((7, 31), 8960), ((7, 32), 33536),
        ((7, 1031), 5915392), ((1000003, -1), 0), ((1000003, 0), 0), ((1000003, 1), 811520), ((1000003, 7), 811520),
        ((1000003, 8), 4325888), ((1000003, 9), 4325888), ((1000003, 31), 4326144), ((1000003, 32), 17302272),
        ((1000003, 1031), 70796032), ((2147483647, -1), 0), ((2147483647, 0), 0), ((2147483647, 1), 811520),
        ((2147483647, 7), 811520), ((2147483647, 8), 4325888), ((2147483647, 9), 4325888), ((2147483647, 31), 4326144),
        ((2147483647, 32), 17302272), ((2147483647, 1031), 70796032),
    ],
    "qk_knn_workspace_bytes": [
        ((-1, 0, 1, 1), 0), ((-1, 1, 1, 1), 0), ((-1, 64, 0, 1), 0), ((-1, 64, 1, 0), 0), ((-1, 64, 1, 1), 0),
        ((-1, 64, 8, 10), 0), ((-1, 64, 9, 10), 0), ((-1, 64, 1024, 256), 0), ((-1, 64, 1, 257), 0),
        ((-1, 4096, 32, 256), 0), ((-1, 4097, 1, 1), 0), ((0, 0, 1, 1), 0), ((0, 1, 1, 1), 256), ((0, 64, 0, 1), 0),
        ((0, 64, 1, 0), 0), ((0, 64, 1, 1), 256), ((0, 64, 8, 10), 256), ((0, 64, 9, 10), 256), ((0, 64, 1024, 256), 256),
        ((0, 64, 1, 257), 0), ((0, 4096, 32, 256), 256), ((0, 4097, 1, 1), 256), ((1, 0, 1, 1), 0), ((1, 1, 1, 1), 768),
        ((1, 64, 0, 1), 0), ((1, 64, 1, 0), 0), ((1, 64, 1, 1), 768), ((1, 64, 8, 10), 1280), ((1, 64, 9, 10), 1280),
        ((1, 64, 1024, 256), 2097408), ((1, 64, 1, 257), 0), ((1, 4096, 32, 256), 65792), ((1, 4097, 1, 1), 768),
        ((1000003, 0, 1, 1), 0), ((1000003, 1, 1, 1), 1792), ((1000003, 64, 0, 1), 0), ((1000003, 64, 1, 0), 0),
        ((1000003, 64, 1, 1), 1792), ((1000003, 64, 8, 10), 84736), ((1000003, 64, 9, 10), 95488),
        ((1000003, 64, 1024, 256), 10486016), ((1000003, 64, 1, 257), 0), ((1000003, 4096, 32, 256), 8651008),
        ((1000003, 4097, 1, 1), 1792), ((2147483647, 0, 1, 1), 0), ((2147483647, 1, 1, 1), 1792),
        ((2147483647, 64, 0, 1), 0), ((2147483647, 64, 1, 0), 0), ((2147483647, 64, 1, 1), 1792),
        ((2147483647, 64, 8, 10), 84736), ((2147483647, 64, 9, 10), 95488), ((2147483647, 64, 1024, 256), 10486016),
        ((2147483647, 64, 1, 257), 0), ((2147483647, 4096, 32, 256), 8651008), ((2147483647, 4097, 1, 1), 1792),
    ],
    "qk_parquet_inflate_workspace_bytes": [
        ((-1,), 0), ((0,), 0), ((1,), 567488), ((3,), 567488), ((4,), 567488), ((5,), 1134976), ((1055,), 149816832),
        ((1056,), 149816832), ((1057,), 149816832), ((1000000,), 149816832),
    ],
}


_QUERY = r"""
import ctypes as C, json, sys
from quokka_b200 import _lib as L
lib = L.lib()
out = {}
for fn, calls in json.load(sys.stdin).items():
    vals = []
    for args in calls:
        if fn == "qk_hashagg_state_bytes":
            desc = L.qk_hashagg_desc()
            desc.capacity, desc.nkeys, desc.nagg = args
            vals.append(lib.qk_hashagg_state_bytes(C.byref(desc)))
        else:
            vals.append(getattr(lib, fn)(*args))
    out[fn] = vals
print(json.dumps(out))
"""


def test_workspace_sizes_are_pinned():
    calls = {fn: [list(args) for args, _ in rows] for fn, rows in PINNED.items()}
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    r = subprocess.run([sys.executable, "-c", _QUERY], input=json.dumps(calls), capture_output=True, text=True, cwd=ROOT,
                       env=env, timeout=600)
    assert r.returncode == 0, r.stderr
    got = json.loads(r.stdout)
    diff = [(fn, args, want, got[fn][i]) for fn, rows in PINNED.items() for i, (args, want) in enumerate(rows) if got[fn][i] != want]
    assert not diff, diff


# ---------------------------------------------------------------- GPU: one byte short
def _short(nbytes, device):
    return torch.empty(max(int(nbytes) - 1, 0), dtype=torch.uint8, device=device)


@pytest.fixture
def short_ws(monkeypatch):
    """ops allocates every kernel workspace one byte short of what qk_*_workspace_bytes asks for."""
    from quokka_b200 import ops
    monkeypatch.setattr(ops, "_ws", _short)
    return ops


def _refused(call):
    from quokka_b200 import ops
    before = ops.launch_count()
    with pytest.raises(L.QkError, match=r"failed \(-4\)"):
        call()
    assert ops.launch_count() == before


def _cases(ops):
    g = torch.Generator().manual_seed(7)
    n, n_by = 100_003, 1000
    key = torch.randint(-1000, 1000, (n,), generator=g, dtype=torch.int64).cuda()
    time = torch.sort(torch.randint(0, 1 << 40, (n,), generator=g, dtype=torch.int64)).values.cuda()
    by = torch.randint(0, n_by, (n,), generator=g, dtype=torch.int32).cuda()
    big = torch.randint(0, 20_000, (n,), generator=g, dtype=torch.int64).cuda()
    x = torch.nn.functional.normalize(torch.randn(n, 64, generator=g), dim=1).cuda()
    vals = torch.rand(n, generator=g, dtype=torch.float64).cuda()
    codes = torch.randint(0, 4, (n,), generator=g, dtype=torch.int32).cuda()
    return {
        "scan_stable": lambda: ops.scan_filter_project([key, vals], [(L.OP_CMP_COL_IMM, 0, L.CMP_LT, 0.0, 500)],
                                                       [[(L.OP_COL, 1, 0, 0.0, 0)]], stable=True),
        "sort": lambda: ops.sort_perm(key, None, False),
        "topk": lambda: ops.topk_candidates(key, 10, True),
        "session_window": lambda: ops.window_session_ids(time, by, 1 << 30),
        "asof_backward": lambda: ops.asof_backward(time, by, time, by, n_by),
        "asof_merge": lambda: ops.asof_merge(time, by, time, by, n_by),
        "partition": lambda: ops.partition_plan(key, 8),
        "partition_radix": lambda: ops.partition_plan(big, 20_000, L.PART_CODE),
        "dense_agg": lambda: ops.DenseAggState([4], [L.AGG_SUM], "cuda").update(
            [codes, vals], None, [0], [[(L.OP_COL, 1, 0, 0.0, 0)]]),
        "gram": lambda: ops.GramState(3, "cuda").update([vals, vals, vals]),     # with or without sums: one plan at k = 3
        "knn": lambda: ops.knn_topk(x, x[:8].contiguous(), 10),
    }


@pytest.mark.gpu
@pytest.mark.parametrize("kernel", ["scan_stable", "sort", "topk", "session_window", "asof_backward", "asof_merge", "partition",
                                    "partition_radix", "dense_agg", "gram", "knn"])
def test_one_byte_short_is_refused_before_any_launch(short_ws, kernel):
    _refused(_cases(short_ws)[kernel])


@pytest.mark.gpu
def test_shift_one_byte_short_is_refused_and_needs_no_workspace_without_a_key(short_ws):
    ops = short_ws
    by = torch.randint(0, 50, (10_007,), dtype=torch.int32).cuda()
    with pytest.MonkeyPatch.context() as m:
        m.setattr(ops, "_ws", lambda nbytes, device: torch.empty(max(int(nbytes), 16), dtype=torch.uint8, device=device))
        dest, seg = ops.partition_plan(by, 50, L.PART_CODE)
    _refused(lambda: ops.shift_plan(1, by.numel(), by, 50, dest, seg))
    src, _, _ = ops.shift_plan(1, by.numel(), device=by.device)
    assert torch.equal(src.cpu(), torch.arange(-1, by.numel() - 1, dtype=torch.int32))


@pytest.mark.gpu
def test_unordered_scan_with_a_short_workspace_runs_the_interpreter():
    """One byte short of qk_scan_workspace_bytes the compaction fast path does not fit, and the unordered scan needs no
    workspace of its own: the filter interpreter runs and finds the same rows."""
    from quokka_b200 import ops
    g = torch.Generator().manual_seed(3)
    n = 1_000_003
    cols = [torch.randint(0, 1000, (n,), generator=g, dtype=torch.int64).cuda(), torch.rand(n, generator=g, dtype=torch.float64).cuda()]
    pred = [(L.OP_CMP_COL_IMM, 0, L.CMP_LT, 0.0, 500)]
    proj = [[(L.OP_COL, 1, 0, 0.0, 0)], [(L.OP_COL, 0, 0, 0.0, 0)]]
    (want_v, want_k), m = ops.scan_filter_project(cols, pred, proj)
    assert ops.last_variant() == "compact_tma"
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(ops, "_ws", _short)
        (v, k), m2 = ops.scan_filter_project(cols, pred, proj)
    assert ops.last_variant() == "filter_interpreter"
    assert m2 == m == int((cols[0] < 500).sum())
    order, want_order = torch.argsort(v), torch.argsort(want_v)         # the interpreter writes the survivors in any order
    assert torch.equal(v[order], want_v[want_order]) and torch.equal(k[order], want_k[want_order])


@pytest.mark.gpu
def test_parquet_inflate_with_a_short_workspace_keeps_fewer_pages_in_flight(tmp_path, monkeypatch):
    """One byte short of qk_parquet_inflate_workspace_bytes is one CTA of slots fewer: the pages still all decode."""
    import pyarrow as pa
    import pyarrow.parquet as pq
    import parquet_cases as P
    from quokka_b200 import ops
    lib = L.lib()
    sizes = []

    def short(n_zstd_pages, device):
        sizes.append(n_zstd_pages)
        return torch.empty(int(lib.qk_parquet_inflate_workspace_bytes(n_zstd_pages)) - 1, dtype=torch.uint8, device=device)

    monkeypatch.setattr(ops, "parquet_inflate_workspace", short)
    rng = np.random.default_rng(11)
    t = pa.table({"a": pa.array(rng.integers(0, 1 << 40, 200_000)), "b": pa.array(rng.random(200_000))})
    for codec in ("zstd", "gzip"):
        path = str(tmp_path / f"{codec}.parquet")
        pq.write_table(t, path, compression=codec, use_dictionary=False, data_page_size=8192)
        P.same(P.read(path, torch.device("cuda", 0)), pq.read_table(path))
    assert sizes and min(sizes) > 8               # at least two CTAs of slots, so one byte short leaves at least one
