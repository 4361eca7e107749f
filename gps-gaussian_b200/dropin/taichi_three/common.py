"""First-call-only initialisation shared by the stand-in's scene objects, and its refusal of unsupported API."""
import os
import sys

_REPO = os.path.dirname(os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))


def repo_on_path():
    """Make `gps_gaussian_b200` importable (the stand-in is found through dropin/ alone)."""
    if _REPO not in sys.path:
        sys.path.insert(0, _REPO)


class Unsupported(NotImplementedError, AttributeError):
    """Raised for reference API the stand-in does not provide.  Also an AttributeError, so `hasattr` stays usable."""


def unsupported(what):
    return Unsupported(f"taichi_three stand-in (gps-gaussian_b200/dropin/taichi_three): {what} is not supported; only the "
                       "API prepare_data/render_data.py uses is provided")


class AutoInit:
    """`init()` runs `_init()` on its first call only (per object); `_init()` may also be called directly to re-run it."""

    def init(self):
        if getattr(self, "_t3_initialised", False):
            return
        self._init()
        self._t3_initialised = True
