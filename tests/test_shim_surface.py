"""tests/cpu_shim.py stands in for every kernel wrapper of quokka_b200.ops: a public function or class of ops that the shim
lacks would surface as an AttributeError inside some executor, in whichever CPU test reaches it first."""
import inspect

import cpu_shim
from quokka_b200 import ops

NO_CPU_MEANING = {"col", "cols"}                    # ctypes descriptors of device tensors for the C ABI


def test_cpu_shim_covers_ops():
    public = sorted(n for n, v in vars(ops).items() if not n.startswith("_") and (inspect.isfunction(v) or inspect.isclass(v))
                    and v.__module__ == ops.__name__)
    print("ops without a CPU meaning, not in cpu_shim:", sorted(NO_CPU_MEANING))
    assert NO_CPU_MEANING <= set(public)
    assert [n for n in public if n not in NO_CPU_MEANING and not hasattr(cpu_shim, n)] == []
