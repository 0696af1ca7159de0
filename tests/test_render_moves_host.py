"""CPU: rendering moved objects per sample -- the rule restated by oracle/render_moves_oracle.py on hand-built rows (identity and
absent moves, take, vacate, rest drop, the air clause, the vacate bounded by the box, the target's view direction), the argument
checks of objects.render_moves and render_rays(moves=), and the ctypes mirror of dmnerf_render_moves (no GPU)."""
import ctypes
import os
import subprocess

import numpy as np
import pytest
import torch

from dmnerf_b200 import _lib
from dmnerf_b200 import objects as OB
from oracle import edit_sweep_oracle as ES
from oracle import render_moves_oracle as RM

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXT = (4.0, 4.0, 4.0)
DIM = 33                                             # grid points and 0.125 steps are exact in fp32
T = np.eye(4)
LEVEL, VOXEL = 0.45, np.float32(11.0 / 128)
C = 4 + 4                                            # ins_num 3
MV, OTHER = 1, 2


def _logits(label):
    row = np.full(C - 4, -4.0, dtype=np.float32)
    row[label] = 4.0
    return row


def _row(label, sigma, colour=0.0):
    return np.concatenate([np.full(3, colour, dtype=np.float32), [np.float32(sigma)], _logits(label)]).astype(np.float32)


def _field(solid):
    """A scene as a function of the point: label MV, sigma 50 where solid(p), else label OTHER and sigma 0; the colour channels
    carry the point and direction so that a taken row shows where it came from."""
    def rows(t, dirs):
        t, dirs = np.asarray(t, dtype=np.float32), np.asarray(dirs, dtype=np.float32)
        out = np.stack([_row(MV, 50.0) if solid(p) else _row(OTHER, 0.0) for p in t]) if len(t) else np.zeros((0, C), np.float32)
        out[:, 0:3] = t
        out[:, 4 + 3] = dirs[:, 0]                   # the last logit (label 3, never the max) carries the direction's x
        return torch.from_numpy(out)
    return rows


def _rays_along_x(ys, zs, depths):
    """Rays along +x through (-2, y, z), depths exact in fp32 -> (rays_o, rays_d, z)."""
    o = np.array([[-2.0, y, z] for y in ys for z in zs], dtype=np.float32)
    d = np.tile(np.array([[1.0, 0.0, 0.0]], dtype=np.float32), (len(o), 1))
    return o, d, np.tile(np.asarray(depths, dtype=np.float32), (len(o), 1))


def _raw(field, o, d, z):
    pts = (o[:, None, :] + d[:, None, :] * z[..., None]).reshape(-1, 3)
    dirs = np.repeat(d / np.linalg.norm(d, axis=1, keepdims=True), z.shape[1], axis=0)
    return field(pts, dirs).reshape(z.shape[0], z.shape[1], C)


def _translate(v):
    m = np.eye(4)
    m[:3, 3] = v
    return m


def _box_of(lo, hi):
    """The inclusive index box of the network-frame corner points lo, hi (identity transform: index = (p + 2) * 8, axes swapped
    (x, y, z) -> (x, -z, y))."""
    inv, b = ES.grid_index_map(T, EXT, DIM)
    q = np.rint(ES.index_of(inv, b, np.array([lo, hi], dtype=np.float32)))
    return tuple(int(v) for a in range(3) for v in (min(q[:, a]), max(q[:, a])))


def _move(label, trans, box, piece=None, rest_drop=False):
    return {"label": label, "trans": trans, "box": box, "piece": piece, "rest_drop": rest_drop}


CUBE = lambda p: bool(np.all(np.abs(p - np.array([-1.0, 0.0, 0.0])) <= 0.25))      # a small cube around (-1, 0, 0)
DEPTHS = np.arange(0.0, 4.0, 0.125, dtype=np.float32)


def _apply(raw, o, d, z, moves, field):
    return RM.apply_moves(raw, o, d, z, moves, T, EXT, DIM, field, LEVEL, VOXEL)


# ---- the rule ---------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("piece_keeps", [None, "all"])
def test_identity_move_changes_nothing(piece_keeps):
    field = _field(CUBE)
    o, d, z = _rays_along_x([0.0, 0.125], [0.0, -0.125], DEPTHS)
    raw = _raw(field, o, d, z)
    piece = None
    if piece_keeps:
        bits = np.full((DIM ** 3 + 31) // 32, 0xFFFFFFFF, dtype=np.uint32)
        piece = ES.Piece(bits, DIM, np.asarray([[8, 0, 0, 16], [0, 0, -8, 16], [0, 8, 0, 16]], dtype=np.float32), True)
    box = _box_of((-1.5, -0.5, -0.5), (-0.5, 0.5, 0.5))
    out, ev = _apply(raw, o, d, z, [_move(MV, np.eye(4), box, piece)], field)
    assert ev > 0
    assert torch.equal(out, raw)


def test_absent_label_and_empty_box_evaluate_nothing():
    field = _field(CUBE)
    o, d, z = _rays_along_x([0.0], [0.0], DEPTHS)
    raw = _raw(field, o, d, z)
    out, ev = _apply(raw, o, d, z, [_move(MV, _translate([1.0, 0.0, 0.0]), ES.EMPTY_BOX)], field)
    assert ev == 0 and torch.equal(out, raw)


def test_translation_takes_the_target_and_vacates_the_source():
    """The cube at x = -1 moved by +1.5 (the scene shows at p what the network holds at p - 1.5): it appears around x = 0.5 and
    its old place is vacated (density 0, logits kept)."""
    field = _field(CUBE)
    o, d, z = _rays_along_x([0.0], [0.0], DEPTHS)
    raw = _raw(field, o, d, z)
    box = _box_of((-1.25, -0.25, -0.25), (-0.75, 0.25, 0.25))
    out, ev = _apply(raw, o, d, z, [_move(MV, _translate([-1.5, 0.0, 0.0]), box)], field)
    x = o[0, 0] + DEPTHS
    new = (np.abs(x - 0.5) <= 0.25)
    old = (np.abs(x + 1.0) <= 0.25)
    r = out[0].numpy()
    assert ev == int(new.sum())
    assert np.all(r[new, 3] == 50.0) and np.all(np.argmax(r[new, 4:], -1) == MV)
    assert np.array_equal(r[new, 0], x[new] - np.float32(1.5))                  # the row comes from the target
    assert np.all(r[old, 3] == 0.0) and np.all(np.argmax(r[old, 4:], -1) == MV)  # vacated, label kept
    rest = ~new & ~old
    assert np.array_equal(r[rest], raw[0].numpy()[rest])


def test_air_clause_keeps_a_solid_sample_under_an_airy_target():
    """A target of the moved label with occ <= level does not replace a solid sample of another label (it would make a hole)."""
    def solid(p):
        return CUBE(p)
    base = _field(solid)

    def field(t, dirs):
        rows = base(t, dirs)
        hit = torch.from_numpy(np.array([CUBE(p) for p in np.asarray(t)], dtype=bool))
        rows[hit, 3] = 0.001                                        # the moved label is air inside the cube
        return rows
    o, d, z = _rays_along_x([0.0], [0.0], DEPTHS)
    raw = _raw(base, o, d, z)
    x = o[0, 0] + DEPTHS
    wall = np.abs(x - 0.5) <= 0.25
    raw[0, torch.from_numpy(wall), 3] = 50.0
    raw[0, torch.from_numpy(wall), 4:] = torch.from_numpy(_logits(OTHER))
    box = _box_of((-1.25, -0.25, -0.25), (-0.75, 0.25, 0.25))
    out, _ = _apply(raw, o, d, z, [_move(MV, _translate([-1.5, 0.0, 0.0]), box)], field)
    assert torch.equal(out[0, torch.from_numpy(wall)], raw[0, torch.from_numpy(wall)])


def test_vacate_is_bounded_by_the_box_and_has_no_level_test():
    """Haze of the moved label (occ below the level) inside the box is vacated too; the label's samples outside the box stay."""
    def field(t, dirs):
        rows = _field(CUBE)(t, dirs)
        t = np.asarray(t)
        haze = torch.from_numpy((np.abs(t[:, 0] - 0.5) <= 0.25) | (np.abs(t[:, 0] + 1.4) <= 0.1))
        rows[haze, 3] = 0.01
        rows[haze, 4:] = torch.from_numpy(_logits(MV))
        return rows
    o, d, z = _rays_along_x([0.0], [0.0], DEPTHS)
    raw = _raw(field, o, d, z)
    box = _box_of((-1.5, -0.25, -0.25), (-0.75, 0.25, 0.25))
    out, _ = _apply(raw, o, d, z, [_move(MV, _translate([-3.0, 0.0, 0.0]), box)], field)
    x = o[0, 0] + DEPTHS
    r, r0 = out[0].numpy(), raw[0].numpy()
    inside = (np.abs(x + 1.0) <= 0.25) | (np.abs(x + 1.4) <= 0.1)
    assert np.all(r[inside, 3] == 0.0)
    far_haze = np.abs(x - 0.5) <= 0.25                              # the label's haze outside the box is not the moved object
    assert np.array_equal(r[far_haze], r0[far_haze])


@pytest.mark.parametrize("rest_drop", [False, True])
def test_rest_drop_vacates_the_label_outside_the_piece(rest_drop):
    """Two cubes of one label; the piece keeps the first only.  The rest (the second cube) is vacated only with rest_drop."""
    second = lambda p: bool(np.all(np.abs(p - np.array([1.0, 0.0, 0.0])) <= 0.25))
    field = _field(lambda p: CUBE(p) or second(p))
    o, d, z = _rays_along_x([0.0], [0.0], DEPTHS)
    raw = _raw(field, o, d, z)
    keep = np.zeros((DIM,) * 3, dtype=bool)
    keep[: DIM // 2] = True                                          # index i < 16: x < 0 keeps the first cube
    vmap = np.asarray([[8, 0, 0, 16], [0, 0, -8, 16], [0, 8, 0, 16]], dtype=np.float32)
    piece = ES.Piece(RO_pack(keep), DIM, vmap, False)
    box = _box_of((-1.25, -0.25, -0.25), (-0.75, 0.25, 0.25))
    out, _ = _apply(raw, o, d, z, [_move(MV, _translate([0.0, 0.0, 0.0]) @ np.eye(4), box, piece, rest_drop)], field)
    x = o[0, 0] + DEPTHS
    sec = np.abs(x - 1.0) <= 0.25
    r = out[0].numpy()
    assert np.all(r[sec, 3] == (0.0 if rest_drop else 50.0))


def RO_pack(mask):
    from oracle import region_oracle as RO
    return RO.pack(mask)


def test_target_direction_is_rotated_and_normalised():
    turn = np.array([[0.0, -1.0, 0.0], [1.0, 0.0, 0.0], [0.0, 0.0, 1.0]])
    d = np.array([[2.0, 0.0, 0.0], [0.0, 3.0, 4.0], [1.0, 1.0, 1.0]], dtype=np.float32)
    got = RM.target_dirs(turn, d)
    assert got.dtype == np.float32
    assert np.array_equal(got[0], np.array([0.0, 1.0, 0.0], dtype=np.float32))
    assert np.array_equal(got[1], np.array([-0.6, 0.0, 0.8], dtype=np.float32))
    n = np.float32(np.sqrt(np.float32(3.0)))
    assert np.array_equal(got[2], np.array([-1.0, 1.0, 1.0], dtype=np.float32) / n)
    # the identity gives the prologue's own d / |d|
    assert np.array_equal(RM.target_dirs(np.eye(3), d), (d / np.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2])[:, None]))


# ---- argument checks ----------------------------------------------------------------------------------------------------------

def _grid():
    return torch.zeros((DIM,) * 3), torch.zeros((DIM,) * 3, dtype=torch.int16)


@pytest.mark.parametrize("kw, msg", [
    (dict(moves=[]), "give between 1 and 8 moves"),
    (dict(moves=[(1, np.eye(4))] * 9), "at most 8 moves"),
    (dict(moves=[(128, np.eye(4))]), "label 128 outside"),
    (dict(moves=[(1, np.diag([1.0, 1.0, -1.0, 1.0]))]), "non-positive determinant"),
    (dict(moves=[(1, np.full((4, 4), np.nan))]), "finite 4x4"),
    (dict(level=1.0), "level 1.0 outside"),
    (dict(rest="sometimes"), "rest must be"),
    (dict(margin=-1), "margin must be"),
    (dict(near=4.0, far=4.0), "must be finite and > 0"),
    (dict(N_importance=0), "must be finite and > 0"),
    (dict(boxes=[[0, DIM, 0, 1, 0, 1]]), "inverted or outside the grid"),
    (dict(boxes=[[0, 1, 0, 1]]), "boxes must be [1, 6]"),
    (dict(pieces=[None, None]), "2 entries for 1 moved labels"),
    (dict(pieces=["region"]), "must be an objects.Region"),
])
def test_render_moves_rejects(kw, msg):
    occ, labels = _grid()
    args = dict(moves=[(1, np.eye(4))])
    args.update(kw)
    with pytest.raises(ValueError) as e:
        OB.render_moves(occ, labels, T, extents=EXT, **args)
    assert msg in str(e.value)


def test_render_rays_rejects_moves_that_are_not_a_moved_scene():
    from dmnerf_b200.render import _check_moved
    with pytest.raises(ValueError, match="render_moves"):
        _check_moved([(1, np.eye(4))], "render_rays", "cpu", None, None)


def test_moved_scene_is_immutable():
    d = _lib.RenderMoves()
    ms = OB.MovedScene(d, (), torch.device("cpu"), (1,), np.zeros((1, 6), dtype=np.int64), [False], 0.45, 0.1)
    with pytest.raises(AttributeError):
        ms.labels = (2,)
    assert ms.abi() is d and ms.boxes == ((0, 0, 0, 0, 0, 0),)


# ---- the C ABI ---------------------------------------------------------------------------------------------------------------------

def test_render_moves_struct_matches_its_ctypes_mirror(tmp_path):
    cls = _lib.RenderMoves
    lines = ['  printf("sizeof %zu\\n", sizeof(dmnerf_render_moves));']
    lines += ['  printf("%s %%zu\\n", offsetof(dmnerf_render_moves, %s));' % (f[0], f[0]) for f in cls._fields_]
    src = tmp_path / "layout.c"
    src.write_text("#include <stddef.h>\n#include <stdio.h>\n#include \"dmnerf_b200.h\"\nint main(void) {\n%s\n  return 0;\n}\n"
                   % "\n".join(lines))
    exe = str(tmp_path / "layout")
    subprocess.run(["cc", "-std=c11", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", exe], check=True)
    got = dict((line.split()[0], int(line.split()[1])) for line in
               subprocess.run([exe], capture_output=True, text=True, check=True).stdout.splitlines())
    want = {"sizeof": ctypes.sizeof(cls)}
    want.update({f[0]: getattr(cls, f[0]).offset for f in cls._fields_})
    assert got == want
    args = _lib.PROTOTYPES["dmnerf_render_moved"][1]
    assert args[7] is ctypes.POINTER(_lib.RenderMoves) and args[8] is ctypes.POINTER(ctypes.c_int64)
