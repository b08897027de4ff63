"""TEST-ONLY numpy restatement of quokka_b200.ops.XchgChannel (csrc/exchange.cu, the K6 shuffle's four channel calls), part
of tests/cpu_shim.py, so that the in-process link (tests/inproc_link.py) and runtime.Exchange's link path run without a GPU.

Control blocks and mailboxes are the same raw memory the kernels address (here: a CPU tensor's), read and written through
numpy views in the `struct XchgCtrl` layout of inproc_link.  The host-side limits of the C ABI are enforced as there --
world / rank / epoch / control-block alignment, at most QK_XCHG_MAX_BUFS buffers, offsets inside the mailbox, element-width
alignment, rows that fit, push_scatter refusing vector and f16 columns, 16-byte aligned recv offsets and outputs -- and a
wait whose flags are missing sets the error word, as the kernel would once its deadline passed."""
from __future__ import annotations

import ctypes

import numpy as np
import torch

import inproc_link as IL
from quokka_b200 import _lib as L

_NP = {torch.uint8: np.uint8, torch.int32: np.int32, torch.int64: np.int64, torch.float32: np.float32,
       torch.float64: np.float64, torch.float16: np.float16}


def _raw(ptr: int, nbytes: int) -> np.ndarray:
    return np.ctypeslib.as_array((ctypes.c_uint8 * int(nbytes)).from_address(int(ptr)))


def _check_rows_col(t: torch.Tensor, who: str):
    """csrc/common.cuh check_rows_col"""
    if t.dtype not in _NP:
        raise L.QkError(f"{who}: bad dtype {t.dtype}")
    if t.dim() == 2 and t.shape[1] > L.KNN_MAX_DIM:
        raise L.QkError(f"{who}: lanes {t.shape[1]} out of range")


def _row_bytes(t: torch.Tensor) -> int:
    return t.element_size() * (t.shape[1] if t.dim() == 2 and t.shape[1] > 1 else 1)


def _rows(t: torch.Tensor) -> np.ndarray:
    """The column as [rows][row bytes] uint8."""
    return t.contiguous().numpy().view(np.uint8).reshape(t.shape[0], _row_bytes(t))


class XchgChannel:
    META = L.XCHG_META_WORDS

    def __init__(self, world, rank, ctrl_ptrs, mailbox_ptrs, mailbox_bytes, device, timeout_ms=30000):
        self.world, self.rank, self.device, self.mailbox_bytes = int(world), int(rank), device, int(mailbox_bytes)
        self.ctrl_ptrs, self.mailbox_ptrs = [int(p) for p in ctrl_ptrs], [int(p) for p in mailbox_ptrs]
        self.epoch = 0

    # ------------------------------------------------------------------ memory
    def _ctrl(self, p: int):
        return IL.ctrl_view(_raw(self.ctrl_ptrs[p], IL.CTRL_USED))

    def _mailbox(self, p: int) -> np.ndarray:
        return _raw(self.mailbox_ptrs[p], self.mailbox_bytes)

    def _chan(self, who: str, epoch: int):
        """fill_chan"""
        if not (1 <= self.world <= L.MAX_PEERS) or not (0 <= self.rank < self.world):
            raise L.QkError(f"{who}: bad world / rank")
        if epoch == 0:
            raise L.QkError(f"{who}: epochs start at 1")
        for p in range(self.world):
            if not self.ctrl_ptrs[p] or self.ctrl_ptrs[p] & 15:
                raise L.QkError(f"{who}: control block of rank {p} missing / misaligned")

    def _wait(self, kind: str, code: int):
        """A wait kernel: the flags of every peer must be there; otherwise its deadline passes and it sets the error word."""
        mine = self._ctrl(self.rank)
        flags = mine.meta_flag if kind == "meta" else mine.data_flag
        if any(int(flags[t]) < self.epoch for t in range(self.world)):
            mine.err[0] = np.uint64((self.epoch << 8) | code)

    def _release(self, kind: str):
        for p in range(self.world):
            c = self._ctrl(p)
            (c.meta_flag if kind == "meta" else c.data_flag)[self.rank] = np.uint64(self.epoch)

    # ------------------------------------------------------------------ the four calls
    def meta(self, words, part_offsets=None):
        if len(words) > self.META:
            raise L.QkError("exchange: too many meta words")
        self.epoch += 1
        self._chan("qk_xchg_meta", self.epoch)
        row = IL.meta_row(self.world, words, part_offsets)
        par = self.epoch & 1
        for p in range(self.world):
            self._ctrl(p).meta[par, self.rank] = row
        self._release("meta")
        self._wait("meta", 1)
        mine = self._ctrl(self.rank)
        if int(mine.err[0]) != 0:
            raise L.QkError(f"exchange: a wait for a peer timed out (status {int(mine.err[0]):#x}): a rank died or fell behind")
        return mine.meta[par, :self.world].copy()

    def _fill(self, who, columns, dst_byte_off, vectors_ok):
        """fill_push: the columns and their destination offsets"""
        n = len(columns)
        if n > L.XCHG_MAX_BUFS:
            raise L.QkError(f"{who}: ncols out of range ({n} buffers, at most {L.XCHG_MAX_BUFS})")
        nrows = columns[0].shape[0] if n else 0
        for c, t in enumerate(columns):
            _check_rows_col(t, who)
            if not vectors_ok and t.dim() == 2 and t.shape[1] > 1:
                raise L.QkError(f"{who}: vector columns are not supported here")
            if not vectors_ok and t.dtype == torch.float16:
                raise L.QkError(f"{who}: f16 elements are only supported in vector columns")
            if t.shape[0] != nrows:
                raise L.QkError(f"{who}: column {c} length mismatch")
        offs = [[int(x) for x in row] for row in dst_byte_off]
        for p in range(self.world):
            if not self.mailbox_ptrs[p]:
                raise L.QkError(f"{who}: mailbox of rank {p} missing")
            for c, t in enumerate(columns):
                o = offs[p][c]
                if o < 0 or o > self.mailbox_bytes:
                    raise L.QkError(f"{who}: offset {o} outside the mailbox ({self.mailbox_bytes} bytes)")
                if o % t.element_size():
                    raise L.QkError(f"{who}: misaligned destination offset")
        return nrows, offs

    def push(self, columns, send_lo, send_hi, dst_byte_off):
        who = "qk_xchg_push"
        self._chan(who, self.epoch)
        nrows, offs = self._fill(who, columns, dst_byte_off, True)
        ranges = []
        for p in range(self.world):
            lo, hi = (int(send_lo[p]), int(send_hi[p])) if columns else (0, 0)
            if lo < 0 or hi < lo or hi > nrows:
                raise L.QkError(f"{who}: bad row range for rank {p}")
            for c, t in enumerate(columns):
                if offs[p][c] + (hi - lo) * _row_bytes(t) > self.mailbox_bytes:
                    raise L.QkError(f"{who}: rows for rank {p} do not fit its mailbox")
            ranges.append((lo, hi))
        for c, t in enumerate(columns):
            src, rb = _rows(t), _row_bytes(t)
            for p, (lo, hi) in enumerate(ranges):
                if hi > lo:
                    self._mailbox(p)[offs[p][c]:offs[p][c] + (hi - lo) * rb] = src[lo:hi].reshape(-1)
        self._release("data")

    def push_scatter(self, columns, dest, part_offsets, dst_byte_off):
        who = "qk_xchg_push_scatter"
        self._chan(who, self.epoch)
        nrows, offs = self._fill(who, columns, dst_byte_off, False)
        if nrows > 0 and (dest is None or part_offsets is None):
            raise L.QkError(f"{who}: null partition plan")
        if nrows > 0:
            d = dest.numpy().astype(np.int64)
            off = part_offsets.numpy().astype(np.int64)
            peer = np.searchsorted(off[1:self.world], d, side="right")     # the kernel's `while (dv >= off[p + 1]) ++p`
            row = d - off[peer]
            for c, t in enumerate(columns):
                src, rb = _rows(t), _row_bytes(t)
                for p in range(self.world):
                    sel = np.nonzero(peer == p)[0]
                    if len(sel):
                        mb = self._mailbox(p)
                        o = offs[p][c]
                        mb[o:o + (len(mb) - o) // rb * rb].reshape(-1, rb)[row[sel]] = src[sel]
        self._release("data")

    def recv(self, src_byte_off, outs):
        who = "qk_xchg_recv"
        self._chan(who, self.epoch)
        if len(outs) > L.XCHG_MAX_BUFS:
            raise L.QkError(f"{who}: ncols out of range ({len(outs)} buffers, at most {L.XCHG_MAX_BUFS})")
        spans = []
        for c, t in enumerate(outs):
            _check_rows_col(t, who)
            nbytes = t.shape[0] * _row_bytes(t)
            o = int(src_byte_off[c])
            if o < 0 or o & 15 or o + nbytes > self.mailbox_bytes:
                raise L.QkError(f"{who}: column {c} lies outside the mailbox or is misaligned")
            if nbytes > 0 and t.data_ptr() & 15:
                raise L.QkError(f"{who}: output {c} is not 16-byte aligned")
            spans.append((o, nbytes))
        self._wait("data", 2)
        mb = self._mailbox(self.rank)
        for t, (o, nbytes) in zip(outs, spans):
            if nbytes:
                t.numpy().view(np.uint8).reshape(-1)[:] = mb[o:o + nbytes]


def install(patch):
    """cpu_shim.install(patch): the rest of the kernels (partition plans, scatter, ...) in numpy on CPU tensors."""
    import cpu_shim                     # cpu_shim imports this module for XchgChannel
    cpu_shim.install(patch)
