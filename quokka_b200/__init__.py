"""quokka_b200 -- H100-native execution backend for Quokka's columnar hot path.

Python mirrors the reference's operator protocols (Executor / input reader / partitioner,
QuokkaContext / DataStream); the work is done by hand-written sm_90a kernels in libqk.so
(include/qk.h).  There is no CPU fallback.

    from quokka_b200 import QuokkaContext
"""
__version__ = "0.1.0"

_LAZY = {
    "QuokkaContext": ("df", "QuokkaContext"),
    "DataStream": ("datastream", "DataStream"),
    "OrderedStream": ("datastream", "OrderedStream"),
    "GroupedDataStream": ("datastream", "GroupedDataStream"),
    "Expression": ("datastream", "Expression"),
    "TaskGraph": ("runtime", "TaskGraph"),
    "DeviceTable": ("columns", "DeviceTable"),
    "TargetInfo": ("target_info", "TargetInfo"),
    "HashPartitioner": ("target_info", "HashPartitioner"),
    "BroadcastPartitioner": ("target_info", "BroadcastPartitioner"),
    "PassThroughPartitioner": ("target_info", "PassThroughPartitioner"),
}


def __getattr__(name):
    """The API classes are resolved on first use so that `import quokka_b200` stays cheap (build scripts,
    `python -m quokka_b200.build`) and does not need torch."""
    if name in _LAZY:
        import importlib
        mod, attr = _LAZY[name]
        return getattr(importlib.import_module(f"{__name__}.{mod}"), attr)
    raise AttributeError(f"module {__name__!r} has no attribute {name!r}")
