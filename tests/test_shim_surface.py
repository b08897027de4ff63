"""tests/cpu_shim.py stands in for every kernel wrapper of quokka_b200.ops, with its signature: a public function or class of
ops that the shim lacks, or a parameter its stand-in does not take, would surface as an AttributeError or TypeError inside
some executor, in whichever CPU test reaches it first."""
import inspect

import cpu_shim
from quokka_b200 import ops

NO_CPU_MEANING = {"col", "cols"}                    # ctypes descriptors of device tensors for the C ABI
NOT_IN_SHIM = {"QuantileSketch.grow"}               # called only from QuantileSketch.update and merge, which the shim states itself


def _public():
    return sorted(n for n, v in vars(ops).items() if not n.startswith("_") and (inspect.isfunction(v) or inspect.isclass(v))
                  and v.__module__ == ops.__name__)


def _methods(cls):
    """{name: function | staticmethod} of the public methods and __init__ that cls itself defines."""
    return {n: v for n, v in vars(cls).items() if (not n.startswith("_") or n == "__init__")
            and (inspect.isfunction(v) or isinstance(v, staticmethod))}


def _params(fn, skip=0):
    """(name, kind, default) of every parameter after the first `skip`."""
    return [(p.name, p.kind.name, p.default) for p in list(inspect.signature(fn).parameters.values())[skip:]]


def test_cpu_shim_covers_ops():
    public = _public()
    print("ops without a CPU meaning, not in cpu_shim:", sorted(NO_CPU_MEANING))
    assert NO_CPU_MEANING <= set(public)
    assert [n for n in public if n not in NO_CPU_MEANING and not hasattr(cpu_shim, n)] == []


def test_functions_take_the_parameters_of_ops():
    bad = [f"{n}: ops {inspect.signature(getattr(ops, n))}, cpu_shim {inspect.signature(getattr(cpu_shim, n))}" for n in _public()
           if inspect.isfunction(getattr(ops, n)) and n not in NO_CPU_MEANING and _params(getattr(ops, n)) != _params(getattr(cpu_shim, n))]
    assert not bad, "\n".join(bad)


def test_methods_take_the_parameters_of_ops():
    """Every public method of every public class of ops and its __init__, `self` left out; a staticmethod must be one in the
    shim too."""
    classes = [n for n in _public() if inspect.isclass(getattr(ops, n))]
    assert all(c in classes and m in _methods(getattr(ops, c)) for c, m in (e.split(".") for e in NOT_IN_SHIM))
    bad = []
    for c in classes:
        for m, want in _methods(getattr(ops, c)).items():
            if f"{c}.{m}" in NOT_IN_SHIM:
                continue
            got = inspect.getattr_static(getattr(cpu_shim, c), m, None)
            if type(got) is not type(want):
                bad.append(f"{c}.{m}: a {type(want).__name__} in ops, {type(got).__name__} in cpu_shim")
                continue
            static = isinstance(want, staticmethod)
            fw, fg, skip = (want.__func__, got.__func__, 0) if static else (want, got, 1)
            if _params(fw, skip) != _params(fg, skip):
                bad.append(f"{c}.{m}: ops {inspect.signature(fw)}, cpu_shim {inspect.signature(fg)}")
    assert not bad, "\n".join(bad)
