"""networks.tester (reference networks/tester.py): `render_test` with the original's signature, printed lines and output files, on
the native renderer and the device-side metrics (dmnerf_b200.tester); lpips, skimage, cv2 and imageio are not needed.
DMNERF_TESTER=reference loads the original's own module from the checkout at DMNERF_REFERENCE_ROOT instead (its imports of
networks.render / networks.helpers still resolve to the native functions through this package)."""
import importlib.util as _ilu
import os as _os

from dmnerf_b200.render import dm_nerf                                     # noqa: F401
from dmnerf_b200.helpers import get_rays_k, z_val_sample                   # noqa: F401
from dmnerf_b200.evaluator import to8b                                     # noqa: F401
from dmnerf_b200.tester import render_test, ins_eval, psnr, ssim           # noqa: F401

_ref = _os.environ.get("DMNERF_REFERENCE_ROOT")
if _os.environ.get("DMNERF_TESTER") == "reference":
    _path = _os.path.join(_ref or "", "networks", "tester.py")
    if not (_ref and _os.path.exists(_path)):
        raise ImportError("DMNERF_TESTER=reference needs DMNERF_REFERENCE_ROOT pointing at a checkout with networks/tester.py")
    _spec = _ilu.spec_from_file_location("_dmnerf_reference_tester", _path)
    _mod = _ilu.module_from_spec(_spec)
    _spec.loader.exec_module(_mod)
    globals().update({k: v for k, v in vars(_mod).items() if not k.startswith("__")})
