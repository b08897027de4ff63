"""The peer-memory shuffle (csrc/exchange.cu, K6) on ONE GPU: W virtual ranks of the in-process link of tests/inproc_link.py
run the same kernel code W GPUs would.  Kernel-level tests compare what every receiver got with numpy, bit for bit --
receiver d gets, from every sender s in rank order, that sender's rows for d in input order -- at the tile edges of
k_xchg_push_scatter (2048-row tiles), with destinations that get nothing, tiles of one destination and a destination that
gets every row, with the contiguous push's segment search over empty ranges, with receive sizes that are not multiples
of 16 bytes, with the meta round's device counts and epoch parity, and with every argument error (which must launch
nothing).  Protocol-level tests run runtime.Exchange on the link (tests/xchg_cases.py, rounds with a small mailbox), and
the hash edge's placement rule is checked against numpy's floor modulo."""
import ctypes as C
import zlib

import numpy as np
import pytest
import torch

import inproc_link as IL
import xchg_cases as XC
from quokka_b200 import _lib as L

pytestmark = pytest.mark.gpu

CUDA = torch.device("cuda")
TILE = 2048                    # csrc/exchange.cu X_TILE


def _ops():
    from quokka_b200 import ops
    return ops


def _al(nbytes: int) -> int:
    return (int(nbytes) + 255) // 256 * 256


def _row_bytes(a: np.ndarray) -> int:
    return a.dtype.itemsize * (a.shape[1] if a.ndim == 2 else 1)


def _dev(a: np.ndarray) -> torch.Tensor:
    return torch.from_numpy(np.ascontiguousarray(a)).to(CUDA)


def _layout(n_recv, cols):
    """Byte offset of every column in a receiver's mailbox (256-byte aligned runs, as runtime.Exchange lays them out)."""
    bases, off = [], 0
    for a in cols:
        bases.append(off)
        off += _al(n_recv * _row_bytes(a))
    return bases, off


def _bits(rng, n, dt):
    """n values of dtype dt with arbitrary bit patterns (NaN payloads, subnormals, negative zero included for floats)."""
    return rng.integers(0, 256, n * np.dtype(dt).itemsize, dtype=np.uint8).view(dt)


def _exchange(link, sends, plan):
    """Runs one exchange of link's W ranks.  sends[s]: sender s's numpy columns; plan(s) -> ("scatter", keys) or
    ("contig", lo[], hi[]).  Returns (received numpy columns per receiver, expected ones)."""
    W, ops = link.world, _ops()
    ncols = len(sends[0])
    picks, devs, words, offs_dev = [], [], [], []
    for s in range(W):
        p = plan(s)
        devs.append([_dev(a) for a in sends[s]])
        if p[0] == "scatter":
            keys = p[1]
            dest, offs = ops.partition_plan(_dev(keys), W, L.PART_MOD)
            part = keys % W
            picks.append([np.nonzero(part == d)[0] for d in range(W)])
            offs_dev.append(offs)
            words.append([-1] * W + [s, 1000 + s])     # words[0:W) are replaced by the device counts
            devs[s] = (devs[s], dest, offs)
        else:
            _, lo, hi = p
            picks.append([np.arange(lo[d], hi[d]) for d in range(W)])
            offs_dev.append(None)
            words.append([hi[d] - lo[d] for d in range(W)] + [s, 1000 + s])
            devs[s] = (devs[s], lo, hi)
    counts = np.array([[len(picks[s][d]) for d in range(W)] for s in range(W)], dtype=np.int64)
    outs = link.meta_round(words, offs_dev)
    assert all(np.array_equal(o[:, :W], counts) for o in outs)
    n_recv = counts.sum(axis=0)
    layout = [_layout(n_recv[d], sends[0]) for d in range(W)]
    assert max(tot for _, tot in layout) <= link.mailbox_bytes
    for s in range(W):
        row0 = counts[:s].sum(axis=0)
        dst = [[layout[d][0][c] + int(row0[d]) * _row_bytes(sends[s][c]) for c in range(ncols)] for d in range(W)]
        cols, a, b = devs[s]
        if isinstance(a, torch.Tensor):
            link.channels[s].push_scatter(cols, a, b, dst)
        else:
            link.channels[s].push(cols, a, b, dst)
    got, exp = [], []
    for d in range(W):
        # outputs pre-filled with 0xA5 bytes: a row the kernels do not deliver shows
        outs = [torch.full((int(n_recv[d]) * _row_bytes(a),), 0xA5, dtype=torch.uint8, device=CUDA)
                .view(torch.from_numpy(a[:0]).dtype).view((int(n_recv[d]),) + a.shape[1:]) for a in sends[0]]
        link.recv(d, layout[d][0], outs)
        got.append([o.cpu().numpy() for o in outs])
        exp.append([np.concatenate([sends[s][c][picks[s][d]] for s in range(W)]) for c in range(ncols)])
    torch.cuda.synchronize()
    assert link.guard_clean(), "a kernel wrote past the last mailbox"
    for r in range(W):
        assert int(link.ctrl(r).err[0]) == 0
    return got, exp


def _assert_same(got, exp, what):
    for d, (g, e) in enumerate(zip(got, exp)):
        for c, (x, y) in enumerate(zip(g, e)):
            assert x.shape == y.shape and np.array_equal(x.view(np.uint8), y.view(np.uint8)), (what, "receiver", d, "column", c)


def _link_for(W, sends):
    """A link whose mailboxes hold every row of every sender (what a broadcast delivers to each receiver)."""
    rows = sum(len(s[0]) for s in sends)
    rb = sum(_row_bytes(a) for a in sends[0])
    return IL.InprocLink(W, rows * rb + 256 * len(sends[0]) + 4096, CUDA, _ops())


# ------------------------------------------------------------------ push_scatter
def _scatter_keys(rng, s, W, n):
    """Sender s's keys (key % W = destination).  With W >= 3 rank W-1 gets nothing; sender s mixes destinations at random
    (s % 3 == 0), sends runs of whole 2048-row tiles to one destination (s % 3 == 1), or sends every row to one
    destination (s % 3 == 2)."""
    active = W - 1 if W >= 3 else W
    mode = s % 3
    if mode == 0:
        d = rng.integers(0, active, n)
    elif mode == 1:
        d = np.repeat(rng.integers(0, active, n // TILE + 1), TILE)[:n]
    else:
        d = np.full(n, (s // 3) % active)
    return d + W * rng.integers(0, 1 << 40, n)


_SCALARS = (np.uint8, np.int32, np.int64, np.float32, np.float64)


@pytest.mark.parametrize("n", [0, 1, 2047, 2048, 2049, 3 * TILE + 5, 1_000_003])
@pytest.mark.parametrize("W", [1, 2, 3, 7, 16])
def test_push_scatter(W, n):
    rng = np.random.default_rng(W * 7919 + n)
    sizes = [n if s % 2 == 0 or n < 2 else n - 1 - s for s in range(W)]          # ragged: the senders' tiles end differently
    keys = [_scatter_keys(rng, s, W, sizes[s]) for s in range(W)]
    sends = [[_bits(rng, sizes[s], dt) for dt in _SCALARS] for s in range(W)]
    link = _link_for(W, sends)
    got, exp = _exchange(link, sends, lambda s: ("scatter", keys[s]))
    _assert_same(got, exp, f"W={W} n={n}")


def test_push_scatter_one_destination_gets_everything():
    W, n = 7, 3 * TILE + 77
    rng = np.random.default_rng(5)
    keys = [3 + W * rng.integers(0, 1 << 40, n) for _ in range(W)]
    sends = [[_bits(rng, n, dt) for dt in _SCALARS] for _ in range(W)]
    got, exp = _exchange(_link_for(W, sends), sends, lambda s: ("scatter", keys[s]))
    assert all(len(g[0]) == 0 for d, g in enumerate(got) if d != 3)
    _assert_same(got, exp, "one destination")


@pytest.mark.parametrize("kind", ["scatter", "contig"])
def test_push_buffer_limit(kind):
    """QK_XCHG_MAX_BUFS buffers in one push (24 columns + 24 validity masks); one more is refused before any launch."""
    W, n = 3, 2 * TILE + 301
    rng = np.random.default_rng(8)
    sends = [[_bits(rng, n, _SCALARS[c % 5]) for c in range(L.XCHG_MAX_BUFS)] for _ in range(W)]
    keys = [rng.integers(0, 1 << 40, n) for _ in range(W)]
    link = _link_for(W, sends)
    plan = (lambda s: ("scatter", keys[s])) if kind == "scatter" else (lambda s: ("contig", [0, 100, 2000], [100, 2000, n]))
    got, exp = _exchange(link, sends, plan)
    _assert_same(got, exp, "max buffers")
    ops, ch = _ops(), link.channels[0]
    cols = [_dev(a) for a in sends[0]] + [_dev(sends[0][0])]
    dst = [[0] * len(cols) for _ in range(W)]
    n0 = ops.launch_count()
    with pytest.raises(L.QkError, match="ncols out of range"):
        if kind == "scatter":
            dest, offs = ops.partition_plan(_dev(keys[0]), W, L.PART_MOD)
            n0 = ops.launch_count()
            ch.push_scatter(cols, dest, offs, dst)
        else:
            ch.push(cols, [0] * W, [n] * W, dst)
    assert ops.launch_count() == n0


# ------------------------------------------------------------------ push (contiguous segments)
def _contig_cols(rng, n):
    return [_bits(rng, n, np.int64), rng.standard_normal((n, 3)).astype(np.float16),           # f16 rows: width 2
            rng.standard_normal((n, 5)).astype(np.float32), rng.integers(0, 256, (n, 7), dtype=np.uint8),
            _bits(rng, n, np.uint8), _bits(rng, n, np.float64)]


@pytest.mark.parametrize("plan", ["broadcast", "single_owner", "grouped"])
@pytest.mark.parametrize("W", [1, 3, 16])
def test_push_contig(W, plan):
    rng = np.random.default_rng(W * 31 + len(plan))
    lo, hi, sends = [], [], []
    for s in range(W):
        if plan == "grouped":
            # every other destination gets an empty range, between non-empty ones (the kernel's tile -> segment search)
            seg = [0 if d % 2 == 1 else int(rng.choice([1, 2047, TILE, 2049, 3 * TILE + 5])) for d in range(W)]
            edges = np.concatenate([[0], np.cumsum(seg)])
            lo.append([int(x) for x in edges[:-1]])
            hi.append([int(x) for x in edges[1:]])
            n = int(edges[-1])
        else:
            n = [0, 1, 2049, 5000, 3 * TILE + 5][s % 5]
            owner = W // 2
            lo.append([0] * W)
            hi.append([n if plan == "broadcast" or d == owner else 0 for d in range(W)])
        sends.append(_contig_cols(rng, n))
    link = _link_for(W, sends)
    got, exp = _exchange(link, sends, lambda s: ("contig", lo[s], hi[s]))
    _assert_same(got, exp, f"{plan} W={W}")


@pytest.mark.parametrize("nbytes", [1, 15, 16, 17, 31, 33, 4095, 4097, 65_537])
def test_recv_byte_tails(nbytes):
    """Receives of byte counts that are not multiples of 16 (k_xchg_copy_out's byte tail), into the front of a larger
    buffer: the bytes after the output stay untouched."""
    W = 2
    rng = np.random.default_rng(nbytes)
    sends = [[rng.integers(0, 256, nbytes, dtype=np.uint8), rng.standard_normal((nbytes, 3)).astype(np.float16)] for _ in range(W)]
    link = _link_for(W, sends)
    b1 = _al(W * nbytes)                  # the f16 rows' column in every receiver's mailbox
    link.meta_round([[nbytes] * W] * W)
    for s in range(W):
        link.channels[s].push([_dev(a) for a in sends[s]], [0] * W, [nbytes] * W, [[s * nbytes, b1 + s * nbytes * 6]] * W)
    for d in range(W):
        big8 = torch.full((W * nbytes + 64,), 0x5A, dtype=torch.uint8, device=CUDA)
        big16 = torch.full((W * nbytes + 8, 3), 7.0, dtype=torch.float16, device=CUDA)
        link.recv(d, [0, b1], [big8[:W * nbytes], big16[:W * nbytes]])
        torch.cuda.synchronize()
        assert np.array_equal(big8[:W * nbytes].cpu().numpy(), np.concatenate([sends[s][0] for s in range(W)]))
        assert np.array_equal(big16[:W * nbytes].cpu().numpy().view(np.uint16), np.concatenate([sends[s][1] for s in range(W)]).view(np.uint16))
        assert bool((big8[W * nbytes:] == 0x5A).all()) and bool((big16[W * nbytes:] == 7.0).all())


# ------------------------------------------------------------------ the meta round
def test_meta_device_counts_override_words():
    W = 5
    rng = np.random.default_rng(3)
    ops = _ops()
    keys = [rng.integers(0, 1 << 40, 10_000 + 17 * s) for s in range(W)]
    offs = [ops.partition_plan(_dev(k), W, L.PART_MOD)[1] for k in keys]
    link = IL.InprocLink(W, 1 << 16, CUDA, ops)
    words = [[-(s + 1) * 1000 - d for d in range(W)] + list(range(s, s + 20)) for s in range(W)]
    outs = link.meta_round(words, offs)
    counts = np.stack([np.bincount(k % W, minlength=W) for k in keys])
    for o in outs:
        assert np.array_equal(o[:, :W], counts)
        assert np.array_equal(o[:, W:W + 20], np.stack([np.arange(s, s + 20) for s in range(W)]))


def test_meta_consecutive_epochs():
    W = 4
    link = IL.InprocLink(W, 1 << 16, CUDA, _ops())
    for e in range(1, 8):
        outs = link.meta_round([[e * 100 + s * 10 + i for i in range(L.XCHG_META_WORDS)] for s in range(W)])
        assert outs[0][W - 1, 0] == e * 100 + (W - 1) * 10


@pytest.mark.parametrize("first_epoch", [1, 2])
@pytest.mark.parametrize("W", [2, 5])
def test_meta_rank_one_round_behind(W, first_epoch):
    """Ranks 0 .. W-2 run meta e and meta e + 1 before rank W-1 runs meta e (what allgather_words and _share_objects'
    trailing meta([0]) create): rank W-1 must still read round e's rows, which the parity double buffer keeps."""
    link = IL.InprocLink(W, 1 << 16, CUDA, _ops())
    if first_epoch == 2:
        link.meta_round([[9] * 3] * W)
    e = link.channels[0].epoch + 1
    words = {ep: [[ep * 1000 + s * 10 + i for i in range(6)] for s in range(W)] for ep in (e, e + 1)}
    rows = {ep: [IL.meta_row(W, words[ep][s]) for s in range(W)] for ep in (e, e + 1)}
    outs = {e: [None] * W, e + 1: [None] * W}
    for ep in (e, e + 1):
        for r in range(W - 1):
            outs[ep][r] = link.meta_turn(r, words[ep][r], None, [(t, rows[ep][t]) for t in range(r + 1, W)])
    for ep in (e, e + 1):
        outs[ep][W - 1] = link.meta_turn(W - 1, words[ep][W - 1])
    for ep in (e, e + 1):
        for r in range(W):
            assert np.array_equal(outs[ep][r], np.stack(rows[ep])), (ep, r)
            link.check_round(r, ep, rows[ep])


# ------------------------------------------------------------------ argument errors: QkError, nothing launched
def test_argument_errors_launch_nothing():
    ops = _ops()
    W, mb = 2, 1 << 16
    link = IL.InprocLink(W, mb, CUDA, ops)
    ch = link.channels[0]
    ch.epoch = 1                                   # as after a meta round, without running one
    x = torch.zeros(10, dtype=torch.int64, device=CUDA)
    d32 = torch.zeros(10, dtype=torch.int32, device=CUDA)
    offs = torch.tensor([0, 10, 10], dtype=torch.int64, device=CUDA)
    host = torch.zeros(W * L.XCHG_META_WORDS + 1, dtype=torch.int64).pin_memory()
    words = (C.c_int64 * L.XCHG_META_WORDS)()

    def raw_meta(world, epoch):
        desc = L.qk_xchg.from_buffer_copy(ch.desc)
        desc.world = world
        L.check(L.lib().qk_xchg_meta(C.byref(desc), epoch, None, words, None, host.data_ptr(), ops._stream()), "qk_xchg_meta")

    misaligned = ops.XchgChannel(W, 0, [link.ctrl_ptrs[0], link.ctrl_ptrs[1] + 8], link.mailbox_ptrs, mb, CUDA, 5000)
    misaligned.epoch = 1
    bad = {
        "world 17": lambda: raw_meta(17, 1),
        "epoch 0": lambda: raw_meta(W, 0),
        "misaligned control block (meta)": lambda: misaligned.meta([1]),
        "misaligned control block (push)": lambda: misaligned.push([x], [0, 0], [10, 10], [[0], [0]]),
        "offset outside the mailbox": lambda: ch.push([x], [0, 0], [10, 10], [[0], [mb + 8]]),
        "rows that do not fit": lambda: ch.push([x], [0, 0], [10, 10], [[0], [mb - 8]]),
        "bad row range": lambda: ch.push([x], [0, 0], [10, 11], [[0], [0]]),
        "misaligned destination offset": lambda: ch.push([x], [0, 0], [10, 10], [[0], [4]]),
        "misaligned destination offset (scatter)": lambda: ch.push_scatter([x], d32, offs, [[0], [4]]),
        "offset outside the mailbox (scatter)": lambda: ch.push_scatter([x], d32, offs, [[0], [mb + 8]]),
        "vector column to push_scatter": lambda: ch.push_scatter([torch.zeros(10, 3, device=CUDA)], d32, offs, [[0], [0]]),
        "f16 column to push_scatter": lambda: ch.push_scatter([torch.zeros(10, dtype=torch.float16, device=CUDA)], d32, offs, [[0], [0]]),
        "too many buffers (recv)": lambda: ch.recv([0] * (L.XCHG_MAX_BUFS + 1), [x] * (L.XCHG_MAX_BUFS + 1)),
        "misaligned recv offset": lambda: ch.recv([8], [torch.empty(4, dtype=torch.int64, device=CUDA)]),
        "recv outside the mailbox": lambda: ch.recv([0], [torch.empty(mb + 1, dtype=torch.uint8, device=CUDA)]),
        "misaligned recv output": lambda: ch.recv([0], [torch.empty(33, dtype=torch.uint8, device=CUDA)[1:]]),
    }
    for what, call in bad.items():
        n0 = ops.launch_count()
        with pytest.raises(L.QkError):
            call()
        assert ops.launch_count() == n0, what
    torch.cuda.synchronize()
    assert not bool(link.buf.any()), "a refused call wrote a flag, a row or the error word"


# ------------------------------------------------------------------ runtime.Exchange on the link
def _exchange_on_link(monkeypatch, world, mailbox_bytes, cases):
    IL.install(monkeypatch)
    from quokka_b200 import runtime as RT
    link = IL.InprocLink(world, mailbox_bytes, CUDA, _ops())

    def rank_body(r):
        ex = RT.Exchange(CUDA)
        cases(ex, CUDA)
        return ex

    exs = IL.run_ranks(link, rank_body)
    torch.cuda.synchronize()
    assert link.guard_clean()
    assert all(int(link.ctrl(r).err[0]) == 0 for r in range(world))
    return exs


@pytest.mark.parametrize("world", [2, 3, 5, 16])
def test_exchange_cases_on_link(monkeypatch, world):
    exs = _exchange_on_link(monkeypatch, world, (16 << 20) + (128 << 20) // world, XC.run_all)
    assert all(ex.peer_calls > 0 for ex in exs)


@pytest.mark.parametrize("world", [2, 5])
def test_exchange_rounds_on_link(monkeypatch, world):
    """A 64 KB mailbox: the payloads go in rounds; the skewed edge makes rounds split again."""
    from quokka_b200 import runtime as RT
    real = RT.Exchange._native_oversize

    def counted(self, *a):          # per Exchange, i.e. per rank thread
        self.depth = getattr(self, "depth", 0) + 1
        self.rounds_entered = getattr(self, "rounds_entered", 0) + 1
        self.max_depth = max(getattr(self, "max_depth", 0), self.depth)
        try:
            return real(self, *a)
        finally:
            self.depth -= 1

    monkeypatch.setattr(RT.Exchange, "_native_oversize", counted)
    exs = _exchange_on_link(monkeypatch, world, 64 << 10, XC.run_rounds)
    assert all(ex.rounds_entered >= 5 for ex in exs), "an edge of run_rounds did not go in rounds"
    assert max(ex.max_depth for ex in exs) >= 2, "no round overflowed a receiver"


# ------------------------------------------------------------------ the hash edge's placement rule
def _placement(keys_dev, nparts, mode=L.PART_MOD):
    """Partition of every row from partition_plan's output, and a check that the plan is the stable grouping."""
    dest, offs = _ops().partition_plan(keys_dev, nparts, mode)
    dest, offs = dest.cpu().numpy().astype(np.int64), offs.cpu().numpy()
    part = np.searchsorted(offs, dest, side="right") - 1
    order = np.argsort(part, kind="stable")
    assert np.array_equal(dest[order], np.arange(len(dest)))
    return part


I64 = np.iinfo(np.int64)


@pytest.mark.parametrize("nparts", [3, 5, 6, 7, 12, 100, 1000, 12_289, 16_383, 16_384])
def test_part_mod_int64_extremes(nparts):
    rng = np.random.default_rng(nparts)
    special = np.array([I64.min, I64.min + 1, I64.min + nparts, -nparts - 1, -nparts, -1, 0, 1, nparts - 1, nparts,
                        I64.max - 1, I64.max, -(1 << 32), -(1 << 32) - 1, (1 << 32), -(1 << 63) + (1 << 32) - 1], dtype=np.int64)
    keys = np.concatenate([special, rng.integers(I64.min, I64.max, 200_000, dtype=np.int64, endpoint=True),
                           rng.integers(-5000, 5000, 50_000)])
    exp = np.array([int(k) % nparts for k in special.tolist()] + list(np.mod(keys[len(special):], nparts)))
    assert np.array_equal(_placement(_dev(keys), nparts), exp)


def _edge_placement(col, n):
    from quokka_b200.columns import DeviceTable
    from quokka_b200.edge import apply_partitioner
    from quokka_b200.target_info import HashPartitioner
    parts = apply_partitioner(HashPartitioner("k"), DeviceTable({"k": col}), 0, n)
    _, dest, offs = parts.pending
    dest, offs = dest.cpu().numpy().astype(np.int64), offs.cpu().numpy()
    return np.searchsorted(offs, dest, side="right") - 1


@pytest.mark.parametrize("n", [2, 3, 7, 16, 100, 16_384])
def test_hash_edge_placement_rule(n):
    import pyarrow as pa
    from quokka_b200.columns import DeviceColumn
    rng = np.random.default_rng(n)
    i32 = np.concatenate([[np.iinfo(np.int32).min, np.iinfo(np.int32).max, -1, 0, 1], rng.integers(-(1 << 31), 1 << 31, 20_000)]).astype(np.int32)
    u8 = np.arange(256, dtype=np.uint8).repeat(7)
    date = np.concatenate([[-719_162, -1, 0, 1, 2_932_896], rng.integers(-30_000, 30_000, 5_000)]).astype(np.int32)   # days since 1970
    for keys, atype in ((i32, None), (u8, None), (date, pa.date32())):
        part = _edge_placement(DeviceColumn(_dev(keys), None, atype), n)
        assert np.array_equal(part, np.mod(keys.astype(np.int64), n)), (keys.dtype, atype)
    f = np.concatenate([[0.0, -0.0, -1.0, 1.0, 5e-324, -5e-324, 2.2250738585072014e-308, -2.2250738585072014e-308,
                         np.inf, -np.inf, np.finfo(np.float64).max, -np.finfo(np.float64).max],
                        rng.standard_normal(10_000) * 1e6, -rng.random(1000) * 1e-310])
    part = _edge_placement(DeviceColumn(_dev(f), None, None), n)
    bits = (f + 0.0).view(np.int64) & np.int64(0x7FFFFFFFFFFFFFFF)
    assert np.array_equal(part, np.mod(bits, n))
    assert part[0] == part[1], "+0.0 and -0.0 land on different ranks"
    words = [f"key-{i}" for i in range(300)]
    codes = rng.integers(0, len(words), 8_000).astype(np.int32)
    part = _edge_placement(DeviceColumn(_dev(codes), words, None), n)
    assert np.array_equal(part, np.array([zlib.crc32(words[c].encode()) % n for c in codes]))


def test_partition_plan_from_two_threads_with_different_part_counts():
    """Two host threads plan partitions at once, into 16 384 parts and into 3: k_part_hist's shared memory grows with the
    part count, and one thread's call must never lower the kernel's limit below what the other's launch needs."""
    import threading
    rng = np.random.default_rng(11)
    keys = rng.integers(I64.min, I64.max, 300_000, dtype=np.int64, endpoint=True)
    errors = []

    def body(nparts):
        try:
            with torch.cuda.stream(torch.cuda.Stream()):
                for _ in range(25):
                    assert np.array_equal(_placement(_dev(keys), nparts), np.mod(keys, nparts)), nparts
        except BaseException as e:          # noqa: B902 -- reported on the test's thread
            errors.append(e)

    threads = [threading.Thread(target=body, args=(n,)) for n in (16_384, 3)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors[0]
