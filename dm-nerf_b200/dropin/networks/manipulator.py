"""networks.manipulator (reference networks/manipulator.py): the edit path runs on the native kernels.  The loops that drive it
(manipulator_eval, manipulator_demo) are the reference's own when DMNERF_REFERENCE_ROOT points at a checkout whose module imports
(lpips, cv2, imageio and skimage installed), with the native functions rebound inside them; otherwise they are the native loops
(dmnerf_b200.manipulator), which need none of those packages."""
import importlib.util as _ilu
import os as _os

_mod = None
_ref = _os.environ.get("DMNERF_REFERENCE_ROOT")
if _ref and _os.path.exists(_os.path.join(_ref, "networks", "manipulator.py")):
    try:
        _spec = _ilu.spec_from_file_location("_dmnerf_reference_manipulator", _os.path.join(_ref, "networks", "manipulator.py"))
        _loaded = _ilu.module_from_spec(_spec)
        _spec.loader.exec_module(_loaded)
        globals().update({k: v for k, v in vars(_loaded).items() if not k.startswith("__")})
        _mod = _loaded
    except ImportError:            # lpips / cv2 / imageio / skimage missing: the native loops below serve instead
        pass

from dmnerf_b200.manipulator import exchanger, manipulator_render, manipulator_nerf, manipulator   # noqa: F401,E402

if _mod is not None:
    # manipulator_eval / manipulator_demo (manipulator.py:208-491) resolve `manipulator`, `exchanger`, ... through the reference
    # module's own globals: rebind them there, otherwise the reference drivers would keep calling the reference torch code.
    from dmnerf_b200.helpers import sample_pdf as _sample_pdf, get_rays_k as _get_rays_k, z_val_sample as _z_val_sample
    for _name, _fn in (("exchanger", exchanger), ("manipulator_render", manipulator_render),
                       ("manipulator_nerf", manipulator_nerf), ("manipulator", manipulator), ("sample_pdf", _sample_pdf),
                       ("get_rays_k", _get_rays_k), ("z_val_sample", _z_val_sample)):
        if hasattr(_mod, _name):
            setattr(_mod, _name, _fn)
else:
    from dmnerf_b200.manipulator import manipulator_eval, manipulator_demo, manipulate_frame   # noqa: F401,E402
