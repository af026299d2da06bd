"""lseg_b200 — H100-native LSeg forward path (drop-in for isl-org/lang-seg's LSegNet.forward).

The directory is named ``lang-seg_b200`` (not an identifier); import it through the top-level
``lseg_b200`` alias module or ``importlib.import_module("lang-seg_b200")``.
"""
from . import _lib  # noqa: F401

__all__ = ["_lib"]
