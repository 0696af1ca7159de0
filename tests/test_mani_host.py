"""CPU: the deformation offsets of the native manipulator_demo against the original's (tests/golden/mani_eval.npz, made by
oracle/make_golden_mani_eval.py from the original loops) and the drop-in resolution of networks.manipulator."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DROPIN = os.path.join(ROOT, "dm-nerf_b200", "dropin")


def test_deform_offsets_equal_the_original_for_every_function(golden_dir):
    from dmnerf_b200.manipulator import deform_offsets, DEFORM_FUNCS
    g = np.load(os.path.join(golden_dir, "mani_eval.npz"))
    objs = json.loads(str(g["demo_deform_objs"]))
    assert sorted(o["deform_func"] for o in objs) == sorted(DEFORM_FUNCS)
    H = int(g["H"])
    ref = g["demo_deform_offsets"]                                        # [view, object, H] float64
    for view in range(ref.shape[0]):
        for j, obj in enumerate(objs):
            got = deform_offsets(obj["deform_func"], H, view)
            assert got.dtype == np.float64 and got.shape == (H,)
            assert np.array_equal(got, ref[view, j]), (obj["deform_func"], view)


def test_sin_deformation_past_its_amplitude_table_is_rejected():
    from dmnerf_b200.manipulator import deform_offsets
    deform_offsets("sin", 16, 7)
    with pytest.raises(ValueError, match="sin"):
        deform_offsets("sin", 16, 8)
    with pytest.raises(ValueError, match="unknown deform_func"):
        deform_offsets("cos", 16, 0)


def _run(code, env_extra, cwd):
    env = {k: v for k, v in os.environ.items() if k != "DMNERF_REFERENCE_ROOT"}
    env.update(env_extra)
    env["PYTHONPATH"] = os.pathsep.join([DROPIN, ROOT])
    return subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, cwd=str(cwd))


_NATIVE = r"""
import sys
import dmnerf_b200.manipulator as nm
import networks.manipulator as M
assert M.manipulator_eval is nm.manipulator_eval and M.manipulator_demo is nm.manipulator_demo
assert M.manipulator is nm.manipulator and M.exchanger is nm.exchanger
assert not {"lpips", "skimage", "cv2", "imageio"} & set(sys.modules)
print("ok")
"""


def test_dropin_serves_the_native_loops_without_a_checkout(tmp_path):
    r = _run(_NATIVE, {}, tmp_path)
    assert r.returncode == 0 and "ok" in r.stdout, r.stderr[-3000:]


def test_dropin_serves_the_native_loops_when_the_checkout_fails_to_import(tmp_path):
    """A checkout whose networks/manipulator.py cannot import (lpips, cv2, imageio or skimage missing)."""
    (tmp_path / "ref" / "networks").mkdir(parents=True)
    (tmp_path / "ref" / "networks" / "manipulator.py").write_text(
        "import lpips_is_not_installed_here\ndef manipulator_eval(*a, **k): return 'original'\n")
    r = _run(_NATIVE, {"DMNERF_REFERENCE_ROOT": str(tmp_path / "ref")}, tmp_path)
    assert r.returncode == 0 and "ok" in r.stdout, r.stderr[-3000:]
