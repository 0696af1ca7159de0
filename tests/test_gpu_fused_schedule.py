"""GPU: the fused render kernel and the RAW-mode training forward return exactly the bits pinned in tests/golden/fused_bits.npz
(oracle/make_golden_fused_bits.py); the selected fused kernels, renders at the instance-head widths and a points-mode query
return those pinned in tests/golden/fused_edge_bits.npz; and a render without the coarse maps (want_coarse=False: the coarse
tile skips its heads) gives the same fine maps, fine depths and fine weights bit for bit as one with them, at every
instance-head width."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from dmnerf_b200 import _lib, synth  # noqa: E402
from oracle import make_golden_fused_bits as G  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
FIXTURE = os.path.join(ROOT, "tests", "golden", "fused_bits.npz")
EDGE_FIXTURE = os.path.join(ROOT, "tests", "golden", "fused_edge_bits.npz")
FINE_KEYS = ("rgb_fine", "depth_fine", "acc_fine", "ins_fine", "z_vals_fine", "weights_fine")


@pytest.fixture(scope="module")
def golden():
    with np.load(FIXTURE) as z:
        return {k: z[k] for k in z.files}


def _check(golden, cases):
    seen = []
    for name, t in cases:
        a = t.detach().cpu().numpy()
        assert name + "#sha256" in golden, "%s: not in the fixture" % name
        assert tuple(a.shape) == tuple(golden[name + "#shape"]) and str(a.dtype) == str(golden[name + "#dtype"]), name
        if not np.array_equal(G.digest(a), golden[name + "#sha256"]):
            got, ref = G.rows(a), golden[name + "#rows"]
            diff = np.abs(got.astype(np.float64) - ref.astype(np.float64))
            pytest.fail("%s differs from the fixture (every %dth row: %d of %d values differ, max abs diff %g)"
                        % (name, G.ROW_STRIDE, int((got != ref).sum()), got.size, float(np.nanmax(diff)) if diff.size else 0.0))
        seen.append(name)
    return seen


def test_fused_renders_match_fixture(golden):
    seen = _check(golden, G.render_cases(DEV))
    expected = [k[:-len("#sha256")] for k in golden if k.endswith("#sha256") and not k.startswith("train/")]
    assert sorted(seen) == sorted(expected)


def test_training_forward_matches_fixture(golden):
    seen = _check(golden, G.train_cases(DEV))
    assert sorted(seen) == ["train/acts", "train/out"]


@pytest.fixture(scope="module")
def edge_golden():
    with np.load(EDGE_FIXTURE) as z:
        return {k: z[k] for k in z.files}


def test_selected_and_head_width_renders_match_fixture(edge_golden):
    seen = _check(edge_golden, G.edge_render_cases(DEV))
    expected = [k[:-len("#sha256")] for k in edge_golden if k.endswith("#sha256") and not k.startswith("points/")]
    assert sorted(seen) == sorted(expected)


def test_points_query_matches_fixture(edge_golden):
    seen = _check(edge_golden, G.points_cases(DEV))
    assert sorted(seen) == ["points/exact/out", "points/f16/out"]


@pytest.mark.parametrize("impl", [_lib.IMPL_UMMA, _lib.IMPL_UMMA_F16], ids=["exact", "fp16"])
@pytest.mark.parametrize("ins_num", [1, 15, 16, 17, 63, 93, 127])
def test_fine_only_render_equals_full(ins_num, impl):
    from dmnerf_b200.render import render_rays
    from dmnerf_b200.testing import make_models
    wl = synth.workload("dmsr_study")
    sel = np.linspace(0, wl["H"] * wl["W"] - 1, 1024).astype(np.int64)
    ro, rd = torch.from_numpy(wl["rays_o"][sel]).to(DEV), torch.from_numpy(wl["rays_d"][sel]).to(DEV)
    z = (torch.linspace(0, 1, 64) * (wl["far"] - wl["near"]) + wl["near"]).to(DEV)
    nc, nf, _, _ = make_models(101, 202, ins_num, DEV)
    with torch.no_grad():
        full = render_rays(ro, rd, nc, nf, z, want_raw=False, want_coarse=True, want_samples=True, impl=impl)
        fine = render_rays(ro, rd, nc, nf, z, want_raw=False, want_coarse=False, want_samples=True, impl=impl)
    assert "rgb_coarse" not in fine
    for k in FINE_KEYS + ("z_vals_coarse",):
        assert torch.equal(fine[k], full[k]), k
