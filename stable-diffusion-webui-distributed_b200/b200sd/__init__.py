"""b200sd — sm_90a (H100) compute path of the local-GPU worker (see DESIGN.md)."""
from . import _lib  # noqa: F401

__all__ = ["_lib"]
