"""networks.manipulator (reference networks/manipulator.py): the edit path runs on the native kernels; the reference's
evaluation / demo loops (manipulator_eval, manipulator_demo: image IO, LPIPS, ...) are re-exported from the reference checkout
when DMNERF_REFERENCE_ROOT points at one and its dependencies are installed."""
import importlib.util as _ilu
import os as _os

_ref = _os.environ.get("DMNERF_REFERENCE_ROOT")
if _ref and _os.path.exists(_os.path.join(_ref, "networks", "manipulator.py")):
    try:
        _spec = _ilu.spec_from_file_location("_dmnerf_reference_manipulator", _os.path.join(_ref, "networks", "manipulator.py"))
        _mod = _ilu.module_from_spec(_spec)
        _spec.loader.exec_module(_mod)
        globals().update({k: v for k, v in vars(_mod).items() if not k.startswith("__")})
    except ImportError:            # lpips / cv2 / imageio / skimage missing: the edit path below does not need them
        pass

from dmnerf_b200.manipulator import exchanger, manipulator_render, manipulator_nerf, manipulator   # noqa: F401,E402

# manipulator_eval / manipulator_demo (manipulator.py:208-491) resolve `manipulator`, `exchanger`, ... through the reference
# module's own globals: rebind them there, otherwise the reference drivers would keep calling the reference torch code.
if "_mod" in globals():
    from dmnerf_b200.helpers import sample_pdf as _sample_pdf, get_rays_k as _get_rays_k, z_val_sample as _z_val_sample
    for _name, _fn in (("exchanger", exchanger), ("manipulator_render", manipulator_render),
                       ("manipulator_nerf", manipulator_nerf), ("manipulator", manipulator), ("sample_pdf", _sample_pdf),
                       ("get_rays_k", _get_rays_k), ("z_val_sample", _z_val_sample)):
        if hasattr(_mod, _name):
            setattr(_mod, _name, _fn)
