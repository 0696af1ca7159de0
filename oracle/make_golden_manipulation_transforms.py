"""Generate tests/golden/mani_transforms.npz from the UNMODIFIED original's generate_poses_eval (tools/pose_generator.py): the
4x4 of each mode (translation, rotation, scale, multi) about each DM-SR scene's manipulation centre.  The function reads the
centre from its own table by args.expname and writes transformation_matrix.json under args.datadir/mani/<mode>/, so it is run
in a temporary directory; the centres are read from the same table (parsed, not imported) and stored beside the matrices.
        python oracle/make_golden_manipulation_transforms.py [CHECKOUT]
CHECKOUT is the original project's checkout (default: $DMNERF_REFERENCE_ROOT)."""
import ast
import os
import sys
import tempfile
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REFERENCE = sys.argv[1] if len(sys.argv) > 1 else os.environ.get("DMNERF_REFERENCE_ROOT")
if not REFERENCE:
    sys.exit("usage: make_golden_manipulation_transforms.py CHECKOUT (or set DMNERF_REFERENCE_ROOT)")
sys.path.insert(0, REFERENCE)
from tools.pose_generator import generate_poses_eval   # noqa: E402

MODES = ("translation", "rotation", "scale", "multi")


def centres():
    """The original's per-scene centre table, read from the source of generate_poses_eval."""
    src = open(os.path.join(REFERENCE, "tools", "pose_generator.py")).read()
    for node in ast.walk(ast.parse(src)):
        if isinstance(node, ast.Assign) and any(getattr(t, "id", None) == "mani_centers" for t in node.targets):
            return ast.literal_eval(node.value)
    raise RuntimeError("mani_centers not found")


def main():
    out = {}
    table = centres()
    with tempfile.TemporaryDirectory() as d:
        for scene, c in sorted(table.items()):
            out[scene + "_centre"] = np.array(c, dtype=np.float64)
            for mode in MODES:
                os.makedirs(os.path.join(d, "mani", mode), exist_ok=True)
                res = generate_poses_eval(types.SimpleNamespace(expname=scene, datadir=d, mani_mode=mode))
                (entry,) = res["transformations"]
                assert entry["mode"] == mode
                out["%s_%s" % (scene, mode)] = np.array(entry["transformation"], dtype=np.float64)
    path = os.path.join(ROOT, "tests", "golden", "mani_transforms.npz")
    np.savez_compressed(path, scenes=np.array(sorted(table)), **out)
    print("wrote", path, len(out), "arrays")


if __name__ == "__main__":
    main()
