"""networks.helpers (reference networks/helpers.py): the hot-path functions come from the native package;
everything else (ray selection for training, rotation helpers) is re-exported from the reference when
DMNERF_REFERENCE_ROOT points at a checkout."""
import importlib.util as _ilu
import os as _os

_ref = _os.environ.get("DMNERF_REFERENCE_ROOT")
if _ref and _os.path.exists(_os.path.join(_ref, "networks", "helpers.py")):
    _spec = _ilu.spec_from_file_location("_dmnerf_reference_helpers", _os.path.join(_ref, "networks", "helpers.py"))
    _mod = _ilu.module_from_spec(_spec)
    _spec.loader.exec_module(_mod)
    globals().update({k: v for k, v in vars(_mod).items() if not k.startswith("__")})

from dmnerf_b200.helpers import sample_pdf, z_val_sample, get_rays_k, get_select_full, get_select_crop   # noqa: F401,E402

# The reference functions re-exported above keep their OWN module globals: rebind the native names inside the loaded
# reference module too, so that every remaining reference helper resolves them to the native versions.
if "_mod" in globals():
    for _name in ("sample_pdf", "z_val_sample", "get_rays_k", "get_select_full", "get_select_crop"):
        setattr(_mod, _name, globals()[_name])
