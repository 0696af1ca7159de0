"""Drop-in `tools` package: `from tools.mesh_generator import mesh_main` (test_dmsr.py:10) resolves to the native mesh extraction
(dmnerf_b200.mesh.mesh_main).  The original's other modules under `tools/` (visualizer, pose_generator) are resolved from the
reference checkout by extending this package's __path__ (DMNERF_REFERENCE_ROOT), as the drop-in `networks` package does."""
import os as _os

_ref = _os.environ.get("DMNERF_REFERENCE_ROOT")
if _ref and _os.path.isdir(_os.path.join(_ref, "tools")):
    __path__.append(_os.path.join(_ref, "tools"))
