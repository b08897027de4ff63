"""The as-of strategy kernels (csrc/asof.cu qk_asof_join, qk_asof_search_join) on the GPU against the numpy statements of
tests/asof_strategy_shim.py, bit for bit -- every strategy, with and without a tolerance (0 included), with carry tables on
both sides, n_by on both sides of the shared-memory table, inputs from empty to several windows per CTA -- a workspace one
byte short refused before any launch, and OrderedStream.join_asof(strategy=...) through the API on the device."""
import ctypes as C
import re

import numpy as np
import pytest
import torch

import asof_strategy_api_cases as A
import asof_strategy_shim as S
import ranks
from quokka_b200 import _lib as L

pytestmark = pytest.mark.gpu

SIZES = ((0, 5), (1, 1), (300, 200), (5000, 7000), (400_000, 1_300_000))
N_BY = (1, 37, 8000, 40_960, 40_961, 70_000)


def _inputs(nl, nr, n_by, seed, span=None):
    rng = np.random.default_rng(seed)
    span = span or max(4, (nl + nr) // 3)                  # heavy ties: ~3 rows per distinct time
    lt = np.sort(rng.integers(-2, span + 2, nl)).astype(np.int64)
    rt = np.sort(rng.integers(0, span, nr)).astype(np.int64)
    return lt, rng.integers(0, n_by, nl).astype(np.int32), rt, rng.integers(0, n_by, nr).astype(np.int32)


def _cuda(*arrays):
    return [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in arrays]


@pytest.mark.parametrize("n_by", N_BY)
@pytest.mark.parametrize("nl,nr", SIZES)
def test_search_join_matches_the_restatement(nl, nr, n_by):
    from quokka_b200 import ops
    lt, lb, rt, rb = _inputs(nl, nr, n_by, nl + n_by)
    args = _cuda(lt, lb, rt, rb)
    for strategy in S.STRATEGIES:
        for tol in (None, 0, 3):
            got = ops.asof_backward(*args, n_by, strategy=strategy, tolerance=tol).cpu().numpy()
            assert np.array_equal(got, S.asof_join(lt, lb, rt, rb, strategy, tol)), (strategy, tol)


@pytest.mark.parametrize("n_by", [n for n in N_BY if n <= 40_960])
@pytest.mark.parametrize("nl,nr", SIZES)
def test_merge_join_matches_the_shim(nl, nr, n_by):
    """Carries on both sides: local rows numbered from r_base = n_by + 5, backward carry rows below it, forward ones past the
    local rows; some keys carry nothing."""
    from quokka_b200 import ops
    lt, lb, rt, rb = _inputs(nl, nr, n_by, 3 * nl + n_by)
    rng = np.random.default_rng(nl + nr)
    r_base = n_by + 5
    cb = np.where(rng.random(n_by) < 0.7, rng.integers(0, r_base, n_by), -1).astype(np.int32)
    cf = np.where(rng.random(n_by) < 0.7, r_base + nr + rng.integers(0, n_by, n_by), -1).astype(np.int32)
    tb = rng.integers(-50, 5, n_by).astype(np.int64)
    tf = (max(rt.max(initial=0), lt.max(initial=0)) + rng.integers(0, 50, n_by)).astype(np.int64)
    args = _cuda(lt, lb, rt, rb)
    dcb, dcf, dtb, dtf = _cuda(cb, cf, tb, tf)
    for strategy in S.STRATEGIES:
        for tol in (None, 0, 3, 60):
            for carried in (False, True):
                kw = dict(strategy=strategy, tolerance=tol)
                back = carried and strategy != "forward"
                fwd = carried and strategy != "backward"
                if fwd:
                    kw.update(carry_fwd=dcf, carry_fwd_time=dtf)
                if back:
                    kw.update(carry_time=dtb)
                want_carry = strategy != "nearest"
                got, carry = ops.asof_merge(*args, n_by, dcb if back else None, r_base, want_carry, **kw)
                exp = S.merge_join(lt, lb, rt, rb, n_by, strategy, tol, cb if back else None, tb, cf if fwd else None, tf, r_base)
                assert np.array_equal(got.cpu().numpy(), exp), (strategy, tol, carried)
                if want_carry:
                    fw = strategy == "forward"
                    ec = S.table_pass(rb, n_by, fw, (cf if fwd else None) if fw else (cb if back else None), r_base)
                    assert np.array_equal(carry.cpu().numpy(), ec), (strategy, tol, carried, "carry_out")


def test_plain_backward_is_unchanged():
    """strategy="backward" without a tolerance through qk_asof_join gives what qk_asof_merge gives."""
    from quokka_b200 import ops
    lt, lb, rt, rb = _inputs(200_000, 600_000, 5000, 11)
    args = _cuda(lt, lb, rt, rb)
    plain, c1 = ops.asof_merge(*args, 5000, want_carry=True)
    huge = 1 << 62                                            # a tolerance that keeps everything
    tol, c2 = ops.asof_merge(*args, 5000, want_carry=True, tolerance=huge)
    assert torch.equal(plain, tol) and torch.equal(c1, c2)
    assert torch.equal(ops.asof_backward(*args, 5000), ops.asof_backward(*args, 5000, tolerance=huge))


def test_workspace_one_byte_short_is_refused():
    from quokka_b200 import ops
    lt, lb, rt, rb = _cuda(*_inputs(3000, 4000, 100, 5))
    out = torch.empty(3000, dtype=torch.int32, device="cuda")
    a, b, c, d = ops.col(lt), ops.col(lb), ops.col(rt), ops.col(rb)
    for strategy in (L.ASOF_BACKWARD, L.ASOF_FORWARD, L.ASOF_NEAREST):
        need = L.lib().qk_asof_join_workspace_bytes(3000, 4000, 100, strategy)
        ws = torch.empty(need, dtype=torch.uint8, device="cuda")
        before = ops.launch_count()
        rc = L.lib().qk_asof_join(C.byref(a), C.byref(b), C.byref(c), C.byref(d), 100, strategy, 2, None, None, None, None, 0, None,
                                  out.data_ptr(), ws.data_ptr(), need - 1, None)
        assert rc == L.ERR_CAPACITY and ops.launch_count() == before
        need = L.lib().qk_asof_workspace_bytes(4000, 100)
        ws = torch.empty(need, dtype=torch.uint8, device="cuda")
        rc = L.lib().qk_asof_search_join(C.byref(a), C.byref(b), C.byref(c), C.byref(d), 100, strategy, 2, out.data_ptr(), ws.data_ptr(),
                                         need - 1, None)
        assert rc == L.ERR_CAPACITY and ops.launch_count() == before
    assert L.lib().qk_asof_join_workspace_bytes(3000, 4000, 100, 7) == 0


@pytest.fixture
def qc():
    from quokka_b200.df import QuokkaContext
    return QuokkaContext()


@pytest.mark.parametrize("case", A.API_CASES, ids=lambda c: c.__name__)
def test_api_case_on_the_device(qc, case, golden_dir):
    import inspect
    args = {"qc": qc, "golden_dir": golden_dir}
    case(*[args[p] for p in inspect.signature(case).parameters])


def test_asof_strategy_two_ranks_nccl():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    rc, out = ranks.torchrun("dist_nccl_asof_strategy_check.py", 2)
    assert rc == 0 and ranks.NCCL_MARKER in out, out[-4000:]
    missing = [n for n in ranks.expand(ranks.SUITES["asof_strategy"]) if not re.search(f"^{re.escape(n)}: ok", out, re.M)]
    assert not missing, f"no ok line for {missing}\n{out[-4000:]}"


def test_merge_join_from_two_threads_with_different_key_counts():
    """Two host threads (two ranks of one process, or two pipeline lanes) run the merge join at once, one with 40 000 keys and
    one with 3: the dynamic shared-memory limit of a kernel is one value for all threads, so one thread's call must never
    lower it below what the other thread's launch needs (csrc/common.cuh raise_smem_limit)."""
    import threading
    from quokka_b200 import ops
    cases = [_inputs(5_000, 20_000, n_by, n_by) + (n_by,) for n_by in (40_000, 3)]
    errors = []

    def body(lt, lb, rt, rb, n_by):
        try:
            args = _cuda(lt, lb, rt, rb)
            exp = S.merge_join(lt, lb, rt, rb, n_by, "backward", None, None, None, None, None, 0)
            with torch.cuda.stream(torch.cuda.Stream()):
                for _ in range(25):
                    got, _ = ops.asof_merge(*args, n_by)
                    assert np.array_equal(got.cpu().numpy(), exp), n_by
        except BaseException as e:          # noqa: B902 -- reported on the test's thread
            errors.append(e)

    threads = [threading.Thread(target=body, args=c) for c in cases]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors[0]
