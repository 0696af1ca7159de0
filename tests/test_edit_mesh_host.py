"""CPU: meshing an edited scene -- the numpy restatement of the rule (oracle/edit_sweep_oracle.py), the vertex-label rule and the
argument checks of the Python layer (no GPU)."""
import ctypes
import os
import subprocess

import numpy as np
import pytest
import torch

from dmnerf_b200 import _lib
from dmnerf_b200 import objects as OB
from oracle import edit_sweep_oracle as E
from oracle import marching_cubes as MC
from oracle import region_oracle as RO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXT = (4.0, 4.0, 4.0)


def _translate(x, y, z):
    m = np.eye(4)
    m[:3, 3] = (x, y, z)
    return m


def _grid(dim, seed, n_labels=4, level=0.45):
    rng = np.random.default_rng(seed)
    occ = rng.random((dim, dim, dim)).astype(np.float32)
    labels = rng.integers(0, n_labels, (dim, dim, dim)).astype(np.int16)
    return occ, labels


def _edit(occ, labels, moves, level=0.45, T=np.eye(4)):
    inv, b = E.grid_index_map(T, EXT, occ.shape[0])
    return E.edit(occ, labels, T, EXT, moves, E.grid_evaluate(occ, labels, inv, b), level)


def test_sweep_points_restate_the_original_grid(golden_dir):
    g = np.load(os.path.join(golden_dir, "mesh_grid.npz"))
    for tag in "ab":
        pts = E.sweep_points(g["transform_" + tag], g["extents"], int(g["dim_" + tag]))
        np.testing.assert_array_equal(pts, g["points_" + tag])


def test_index_map_inverts_the_grid_affine(golden_dir):
    g = np.load(os.path.join(golden_dir, "mesh_grid.npz"))
    for tag in "ab":
        T, dim = g["transform_" + tag], int(g["dim_" + tag])
        A, b = OB.grid_affine(T, dim, g["extents"])
        inv, b2 = E.grid_index_map(T, g["extents"], dim)
        np.testing.assert_allclose(inv, np.linalg.inv(A), rtol=1e-12, atol=1e-12)
        np.testing.assert_allclose(b2, b, rtol=1e-12, atol=1e-12)
        u = E.index_of(inv, b, g["points_" + tag])
        idx = np.stack(np.meshgrid(*[np.arange(dim)] * 3, indexing="ij"), -1).reshape(-1, 3)
        assert np.abs(u - idx).max() < 1e-4


def test_identity_reproduces_the_grid_and_an_absent_label_changes_nothing():
    occ, labels = _grid(9, 3)
    for mv in range(4):
        box = E.solid_box(occ, labels, mv, 0.45, 2)
        o, lab, n = _edit(occ, labels, [dict(label=mv, trans=np.eye(4), box=box)])
        np.testing.assert_array_equal(o, occ)
        np.testing.assert_array_equal(lab, labels)
        assert n > 0
    absent = dict(label=7, trans=_translate(0.5, 0, 0), box=E.solid_box(occ, labels, 7, 0.45, 2))
    assert absent["box"] == E.EMPTY_BOX
    o, lab, n = _edit(occ, labels, [absent])
    assert n == 0
    np.testing.assert_array_equal(o, occ)
    np.testing.assert_array_equal(lab, labels)


def _two_cubes(dim=17):                            # grid points and 0.25 steps are exact in fp32
    occ = np.zeros((dim,) * 3, dtype=np.float32)
    labels = np.zeros((dim,) * 3, dtype=np.int16)
    occ[6:8, 3:5, 3:5] = 0.9
    labels[6:8, 3:5, 3:5] = 1                         # piece A
    occ[2:4, 8:10, 8:10] = 0.8
    labels[2:4, 8:10, 8:10] = 1                       # piece B of the same label
    occ[0:2, 0:2, 0:2] = 0.7
    labels[0:2, 0:2, 0:2] = 2                         # another object
    return occ, labels


def test_a_moved_object_is_vacated_and_lands_at_the_inverse_move():
    occ, labels = _two_cubes()
    # two voxels along the network x (grid index i): the edit shows at p what is at p + 2 voxels, so the object moves to i - 2
    step = EXT[0] / (occ.shape[0] - 1)
    move = dict(label=1, trans=_translate(2 * step, 0, 0), box=(0, 16, 0, 16, 0, 16))
    o, lab, n = _edit(occ, labels, [move])
    assert n == 17 ** 3 - 2 * 17 * 17                 # targets with i + 2 <= 16
    want_o, want_l = occ.copy(), labels.copy()
    want_o[labels == 1] = 0.0                         # vacated, label kept
    want_o[4:6, 3:5, 3:5], want_l[4:6, 3:5, 3:5] = 0.9, 1
    want_o[0:2, 8:10, 8:10], want_l[0:2, 8:10, 8:10] = 0.8, 1
    np.testing.assert_array_equal(o, want_o)
    np.testing.assert_array_equal(lab, want_l)


@pytest.mark.parametrize("rest", ["keep", "drop"])
def test_a_piece_moves_alone_and_the_rest_is_kept_or_dropped(rest):
    occ, labels = _two_cubes()
    dim = occ.shape[0]
    A, b = OB.grid_affine(np.eye(4), dim, EXT)
    mask = np.zeros((dim,) * 3, dtype=bool)
    mask[6:8, 3:5, 3:5] = True
    piece = E.Piece(RO.pack(mask), dim, RO.voxel_map(A, b), outside_keep=True)
    keep = piece.keeps(E.sweep_points(np.eye(4), EXT, dim)).reshape(occ.shape)
    box = E.solid_box(occ, labels, 1, 0.45, 2, keep)
    assert box == (4, 9, 1, 6, 1, 6)
    step = EXT[0] / (dim - 1)
    o, lab, _ = _edit(occ, labels, [dict(label=1, trans=_translate(2 * step, 0, 0), box=box, piece=piece,
                                         rest_drop=rest == "drop")])
    want_o, want_l = occ.copy(), labels.copy()
    want_o[6:8, 3:5, 3:5] = 0.0
    want_o[4:6, 3:5, 3:5], want_l[4:6, 3:5, 3:5] = 0.9, 1
    if rest == "drop":
        want_o[2:4, 8:10, 8:10] = 0.0
    np.testing.assert_array_equal(o, want_o)
    np.testing.assert_array_equal(lab, want_l)


def test_air_of_a_moved_object_does_not_punch_holes():
    occ, labels = _two_cubes()
    step = EXT[0] / (occ.shape[0] - 1)
    # label 2's cube sits at i 0..1; moving label 1's piece B (at i 2..3) two voxels toward it carries label-1 air onto nothing
    # solid, and a solid point of label 0 in the way keeps its value
    occ[0:2, 8:10, 8:10] = 0.95
    o, lab, _ = _edit(occ, labels, [dict(label=1, trans=_translate(2 * step, 0, 0), box=(0, 16, 0, 16, 0, 16))])
    np.testing.assert_array_equal(o[0:2, 8:10, 8:10], np.float32(0.8))          # a solid target wins over a solid point
    labels2 = labels.copy()
    labels2[4:6, 8:10, 8:10] = 1                                                 # label-1 air next to piece B
    occ2 = occ.copy()
    occ2[2:4, 8:10, 8:10] = 0.9
    labels2[2:4, 8:10, 8:10] = 0
    o, lab, _ = _edit(occ2, labels2, [dict(label=1, trans=_translate(2 * step, 0, 0), box=(0, 16, 0, 16, 0, 16))])
    np.testing.assert_array_equal(o[2:4, 8:10, 8:10], np.float32(0.9))          # air does not replace solid
    np.testing.assert_array_equal(lab[2:4, 8:10, 8:10], 0)


def _mc_inside_end_labels(g, labels, level, v):
    """The label of the inside end of each marching-cubes vertex's edge (vertex = p + t e_a)."""
    out = []
    for x in v:
        f = np.floor(x).astype(int)
        frac = x - f
        a = int(np.argmax(frac)) if frac.max() > 0 else None
        if a is None:                                  # on a grid point: that point (inside) or, outside, no unique end
            out.append(int(labels[tuple(f)]) if g[tuple(f)] > level else None)
            continue
        lo, hi = f.copy(), f.copy()
        hi[a] += 1
        out.append(int(labels[tuple(lo)]) if g[tuple(lo)] > level else int(labels[tuple(hi)]))
    return out


def test_vertex_labels_are_the_inside_end_of_each_edge():
    rng = np.random.default_rng(5)
    g = rng.random((9, 8, 7)).astype(np.float32)
    cube = np.zeros((9, 9, 9), dtype=np.float32)
    cube[:9, :8, :7] = g
    labels = rng.integers(0, 6, cube.shape).astype(np.int16)
    v, _, _ = MC.marching_cubes(cube, 0.45)
    got = E.vertex_labels(v, cube, labels, 0.45)
    want = _mc_inside_end_labels(cube, labels, 0.45, v)
    assert all(w is None or w == x for w, x in zip(want, got))
    np.testing.assert_array_equal(got, E.nearest_solid_bruteforce(v, cube, labels, 0.45))


def test_vertex_on_a_grid_point_takes_the_lowest_linear_index():
    g = np.zeros((5, 5, 5), dtype=np.float32)
    labels = np.arange(125, dtype=np.int16).reshape(5, 5, 5)
    g[2, 2, 2] = 0.45                                   # exactly the level: outside, and the crossing t of its edges is 1
    for d in [(-1, 0, 0), (1, 0, 0), (0, -1, 0), (0, 1, 0), (0, 0, -1), (0, 0, 1)]:
        g[2 + d[0], 2 + d[1], 2 + d[2]] = 0.9
    v, _, _ = MC.marching_cubes(g, 0.45)
    on = np.all(v == np.float32(2.0), axis=1)
    assert on.any()                                      # a vertex sits on (2, 2, 2), all six solid neighbours at distance 1
    got = E.vertex_labels(v, g, labels, 0.45)
    assert (got[on] == labels[1, 2, 2]).all()           # the lowest linear index of the six
    np.testing.assert_array_equal(got, E.nearest_solid_bruteforce(v, g, labels, 0.45))
    solid_pt = np.array([[1.0, 2.0, 2.0], [9.0, 9.0, 9.0], [np.nan, 0, 0]], dtype=np.float32)
    np.testing.assert_array_equal(E.vertex_labels(solid_pt, g, labels, 0.45), [labels[1, 2, 2], -1, -1])


def test_python_layer_rejects_bad_arguments():
    from dmnerf_b200.model import DM_NeRF
    net = DM_NeRF(8, 256, 63, 27, [4], 13)
    eye = np.eye(4)
    bad = [
        (dict(moves=[(1, eye)] * 9), "at most 8"),
        (dict(moves=[(14, eye)]), "outside"),
        (dict(moves=[(1, np.full((4, 4), np.nan))]), "finite"),
        (dict(moves=[(1, np.diag([1.0, 1.0, -1.0, 1.0]))]), "determinant"),
        (dict(moves=[(1, np.ones((3, 4)))]), "4x4"),
        (dict(moves=[(1, eye)], level=1.0), "level"),
        (dict(moves=[(1, eye)], boxes=[(0, 9, 0, 8, 0, 8)]), "inverted or outside"),
        (dict(moves=[(1, eye)], boxes=[(3, 2, 0, 1, 0, 1)]), "inverted or outside"),
        (dict(moves=[(1, eye)], rest="gone"), "rest"),
        (dict(moves=[(1, eye)], pieces=[None, None]), "pieces"),
        (dict(moves=[(1, eye)], margin=-1), "margin"),
    ]
    for kw, msg in bad:
        with pytest.raises(ValueError, match=msg):
            OB.edited_sweep(net, eye, grid_dim=9, **kw)
    assert OB.EMPTY_BOX == E.EMPTY_BOX
    assert OB._check_boxes([OB.EMPTY_BOX], 1, 9).tolist() == [list(OB.EMPTY_BOX)]


def test_move_struct_matches_its_ctypes_mirror(tmp_path):
    fields = [f[0] for f in _lib.EditMove._fields_]
    lines = ['  printf("sizeof %zu\\n", sizeof(dmnerf_edit_move));']
    lines += ['  printf("%s %%zu\\n", offsetof(dmnerf_edit_move, %s));' % (f, f) for f in fields]
    src = tmp_path / "layout.c"
    src.write_text("#include <stddef.h>\n#include <stdio.h>\n#include \"dmnerf_b200.h\"\nint main(void) {\n%s\n  return 0;\n}\n"
                   % "\n".join(lines))
    exe = str(tmp_path / "layout")
    subprocess.run(["cc", "-std=c11", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", exe], check=True)
    got = dict((line.split()[0], int(line.split()[1])) for line in
               subprocess.run([exe], capture_output=True, text=True, check=True).stdout.splitlines())
    want = {"sizeof": ctypes.sizeof(_lib.EditMove)}
    want.update({f: getattr(_lib.EditMove, f).offset for f in fields})
    assert got == want
    assert _lib.PROTOTYPES["dmnerf_mesh_occupancy_edit"][1][8] is ctypes.POINTER(_lib.EditMove)
    assert "dmnerf_mesh_vertex_labels" in _lib.PROTOTYPES
