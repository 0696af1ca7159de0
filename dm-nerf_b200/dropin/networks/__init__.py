"""Drop-in `networks` package: put `<repo>/dm-nerf_b200/dropin` (and the repo root) ahead of the reference
checkout on PYTHONPATH and the reference's train_*.py / test_*.py / config.py import the native renderer
through their own, unmodified import lines (`from networks.render import dm_nerf`, ...).  Modules of the
reference's `networks/` that this package does not provide are resolved from the reference checkout by extending this
package's __path__ (DMNERF_REFERENCE_ROOT)."""
import os as _os

_ref = _os.environ.get("DMNERF_REFERENCE_ROOT")
if _ref and _os.path.isdir(_os.path.join(_ref, "networks")):
    __path__.append(_os.path.join(_ref, "networks"))
