"""Imported by Python at start-up when `gps-gaussian_b200/dropin` is on PYTHONPATH.  Does nothing unless GPSG_PATCH=1, in
which case the reference's `core.corr.CorrBlockFast1D` / `lib.GaussianRender.pts2render` are rebound to the fused sm_90a
paths right after the reference imports those modules (see gps_gaussian_b200/patch.py and INTEGRATION.md)."""
import os
import sys

if os.environ.get("GPSG_PATCH", "0") == "1":
    _repo = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    if _repo not in sys.path:
        sys.path.insert(0, _repo)
    from gps_gaussian_b200 import patch as _patch
    _patch.install()

# keep whatever sitecustomize this one shadows (e.g. the distribution's apport hook) working
for _p in sys.path:
    _f = os.path.join(_p or ".", "sitecustomize.py")
    if os.path.isfile(_f) and os.path.abspath(_f) != os.path.abspath(__file__):
        try:
            with open(_f) as _fh:
                exec(compile(_fh.read(), _f, "exec"), {"__name__": "sitecustomize", "__file__": _f})
        except Exception:
            pass
        break
