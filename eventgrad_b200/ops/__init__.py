"""Python front-ends of the sm_90a extension (eventgrad_b200/_C*.so, built by build_ext.py).

`ext()` returns the compiled module.  On a machine with a GPU a missing / unloadable extension
is a hard error -- there is deliberately NO silent PyTorch fallback for the fused ops, so a run
that reports numbers has provably executed the native kernels.
"""
from __future__ import annotations

import importlib
import os

_EXT = None


def ext():
    global _EXT
    if _EXT is not None:
        return _EXT
    try:
        _EXT = importlib.import_module("eventgrad_b200._C")
    except ImportError as e:
        if os.environ.get("EGB_NO_AUTOBUILD") == "1":
            raise
        try:
            from ..build_ext import build
            build()
            _EXT = importlib.import_module("eventgrad_b200._C")
        except Exception as e2:  # noqa: BLE001
            raise ImportError(
                "eventgrad_b200._C (sm_90a extension) is not built and could not be built: "
                f"{e!r} / {e2!r}. Run `python -m eventgrad_b200.build_ext`.") from e2
    return _EXT


def ext_available() -> bool:
    try:
        ext()
        return True
    except ImportError:
        return False
