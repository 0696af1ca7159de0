"""CPU: colouring an edited view (DESIGN.md, "Colouring an edited view") as oracle/edit_view_oracle.py restates it, on hand-built
grids: the provenance replay at every grid point reproduces the grid-only edit (deform_oracle.grid_edit) for a whole-voxel
translation, a quarter turn, two moves where the second overwrites the first, a copy, a group, a piece with the rest kept and
dropped, a deformation and a vacate after a take; the move it names, the colour point and the direction on cast rays; the
consistency check on a grid that is not the edit; and grid_view's argument checks for moves= and source=, which run before any
device work."""
import numpy as np
import pytest
import torch

from dmnerf_b200 import _lib
from dmnerf_b200 import objects as OB
from oracle import deform_oracle as DO
from oracle import edit_sweep_oracle as E
from oracle import edit_view_oracle as EV
from oracle import region_oracle as RO

DIM = 16
EXT = (DIM - 1.0,) * 3                        # one network unit per voxel
C = (DIM - 1) / 2.0
LEVEL = 0.45
FULL = (0, DIM - 1) * 3


def _net(i, j, k):
    """The network point of index (i, j, k) with T = I and EXT: (i - c, -(k - c), j - c)."""
    return np.array([i - C, -(k - C), j - C], dtype=np.float64)


def _translate(di, dj, dk):
    """The move that shows at p the source at p - (di, dj, dk) voxels: the object moves by +(di, dj, dk)."""
    m = np.eye(4)
    m[:3, 3] = -(_net(di, dj, dk) - _net(0, 0, 0))
    return m


def _scene():
    """A floor (label 1), a block (label 3) with a slab on it (label 4) and a post (label 5)."""
    occ = np.zeros((DIM,) * 3, dtype=np.float32)
    lab = np.ones((DIM,) * 3, dtype=np.int16)
    rng = np.random.default_rng(3)

    def put(sl, label):
        occ[sl] = rng.uniform(0.5, 1.0, occ[sl].shape).astype(np.float32)
        lab[sl] = label
    put(np.s_[:, :, 0:1], 1)
    put(np.s_[3:6, 3:6, 1:4], 3)
    put(np.s_[3:6, 3:6, 4:5], 4)
    put(np.s_[10:12, 9:12, 1:6], 5)
    return occ, lab


def _move(label, trans, **kw):
    return dict(label=label, trans=trans, box=kw.pop("box", FULL), **kw)


def _edited(src_occ, src_lab, moves):
    o, l, _, _ = DO.grid_edit(src_occ, src_lab, src_occ, src_lab, np.eye(4), EXT, moves, LEVEL)
    return o, l


def _replay_everywhere(src_occ, src_lab, moves):
    """The provenance of every grid point, checked against the grid-only edit -> (move [dim^3], edited occ, edited labels)."""
    occ, lab = _edited(src_occ, src_lab, moves)
    allv = np.arange(DIM ** 3)
    m, o_r, l_r = EV.provenance(src_occ, src_lab, np.eye(4), EXT, moves, allv, LEVEL)
    assert np.array_equal(o_r.view(np.int32), occ.reshape(-1).view(np.int32))
    assert np.array_equal(l_r, lab.reshape(-1).astype(np.int64))
    assert not EV.mismatched(occ, lab, allv, o_r, l_r).any()
    return m.reshape((DIM,) * 3), occ, lab


def _rays():
    """Rays down every column (-k), along +i and along +j through every voxel centre line, from outside the grid."""
    o, d = [], []
    for a, b in np.ndindex(DIM, DIM):
        o += [_net(a, b, DIM + 1), _net(-2, a, b), _net(a, -2, b)]
        d += [_net(0, 0, -1) - _net(0, 0, 0), _net(1, 0, 0) - _net(0, 0, 0), _net(0, 1, 0) - _net(0, 0, 0)]
    return np.array(o, dtype=np.float32), np.array(d, dtype=np.float32)


def _view(src_occ, src_lab, moves):
    occ, lab = _edited(src_occ, src_lab, moves)
    o, d = _rays()
    r = EV.edit_view(occ, lab, src_occ, src_lab, np.eye(4), EXT, o, d, 0.0, 100.0, moves, LEVEL)
    assert not r["mismatched"].any()
    hit = r["cast"]["voxel"] >= 0
    assert hit.sum() > 100
    assert (r["move"][~hit] == -1).all() and np.isnan(r["point"][~hit]).all() and (r["dir"][~hit] == 0).all()
    with np.errstate(invalid="ignore"):                                     # inf depth times a zero component off hits
        x = (o + (r["cast"]["t"][:, None] * d).astype(np.float32)).astype(np.float32)
    still = hit & (r["move"] < 0)
    assert np.array_equal(r["point"][still], x[still]) and np.array_equal(r["dir"][still], d[still])
    return r, occ, lab, o, d, x


def test_whole_voxel_translation_names_the_move_and_shifts_the_point():
    occ, lab = _scene()
    moves = [_move(3, _translate(6, 0, 0))]
    m, e_occ, e_lab = _replay_everywhere(occ, lab, moves)
    assert ((e_lab == 3) & (e_occ > LEVEL)).sum() == 27
    assert np.array_equal(m == 0, (e_lab == 3) & (e_occ > LEVEL))   # every point of the moved block, and nothing else
    r, _, _, o, d, x = _view(occ, lab, moves)
    moved = r["move"] == 0
    assert moved.sum() > 0 and (r["cast"]["label"][moved] == 3).all()
    shifted = x[moved].copy()
    shifted[:, 0] -= np.float32(6.0)                                         # exact: whole network units
    assert np.array_equal(r["point"][moved], shifted)
    assert np.array_equal(r["dir"][moved], d[moved])


def test_quarter_turn_rotates_the_point_and_the_direction():
    occ, lab = _scene()
    c = _net(4, 4, 2)
    R = np.array([[0.0, -1.0, 0.0], [1.0, 0.0, 0.0], [0.0, 0.0, 1.0]])       # about network z: the grid's -k axis
    trans = np.eye(4)
    trans[:3, :3] = R
    trans[:3, 3] = c - R @ c
    moves = [_move(3, trans)]
    m, e_occ, e_lab = _replay_everywhere(occ, lab, moves)
    assert np.array_equal(m == 0, (e_lab == 3) & (e_occ > LEVEL))
    r, _, _, o, d, x = _view(occ, lab, moves)
    moved = r["move"] == 0
    assert moved.any()
    assert np.array_equal(r["point"][moved], E.targets(trans[:3], x[moved]))
    assert np.array_equal(r["dir"][moved], (d[moved].astype(np.float64) @ R.T).astype(np.float32))


def test_the_second_move_overwrites_the_first():
    occ, lab = _scene()
    moves = [_move(3, _translate(6, 0, 0)), _move(5, _translate(-1, -5, 0))]      # the post lands on the moved block
    m, e_occ, e_lab = _replay_everywhere(occ, lab, moves)
    solid = e_occ > LEVEL
    assert np.array_equal(m == 1, (e_lab == 5) & solid)
    assert np.array_equal(m == 0, (e_lab == 3) & solid)
    assert (m[9:11, 4:6, 1:4] == 1).all() and (e_lab[9:11, 4:6, 1:4] == 5).all()   # placed by the first move, then the second
    r, *_ = _view(occ, lab, moves)
    assert set(np.unique(r["move"][r["cast"]["voxel"] >= 0])) == {-1, 0, 1}


def test_a_copy_leaves_its_source_unattributed():
    occ, lab = _scene()
    moves = [_move(3, _translate(6, 0, 0), copy=True)]
    m, e_occ, e_lab = _replay_everywhere(occ, lab, moves)
    assert (m[3:6, 3:6, 1:4] == -1).all() and (m[9:12, 3:6, 1:4] == 0).all()
    assert ((e_lab == 3) & (e_occ > LEVEL)).sum() == 54


def test_a_group_carries_its_labels_under_one_move():
    occ, lab = _scene()
    moves = [_move(3, _translate(6, 0, 0), group=[3, 4])]
    m, e_occ, e_lab = _replay_everywhere(occ, lab, moves)
    assert (m[9:12, 3:6, 1:5] == 0).all() and (e_lab[9:12, 3:6, 4] == 4).all()
    r, *_ = _view(occ, lab, moves)
    moved = r["move"] == 0
    assert set(np.unique(r["cast"]["label"][moved])) == {3, 4}


@pytest.mark.parametrize("rest_drop", [False, True])
def test_a_piece_with_the_rest_kept_or_dropped(rest_drop):
    occ, lab = _scene()
    keep = np.zeros((DIM,) * 3, dtype=bool)
    keep[:, :4, :] = True                                                    # the block's j = 3 slice is the piece
    inv, b = E.grid_index_map(np.eye(4), EXT, DIM)
    vmap = np.concatenate([inv, (-inv @ b)[:, None]], 1).astype(np.float32)
    piece = E.Piece(RO.pack(keep), DIM, vmap, False)
    moves = [_move(3, _translate(6, 0, 0), piece=piece, rest_drop=rest_drop)]
    m, e_occ, e_lab = _replay_everywhere(occ, lab, moves)
    assert (m[9:12, 3, 1:4] == 0).all() and (m[9:12, 4:6, 1:4] == -1).all()
    rest = e_occ[3:6, 4:6, 1:4] > LEVEL
    assert (not rest.any()) if rest_drop else rest.all()
    assert (m[3:6, 4:6, 1:4] == -1).all()


def test_a_deformation_pulls_the_point_and_the_direction_back():
    occ, lab = _scene()
    up = _net(0, 0, 1) - _net(0, 0, 0)
    d = OB.deformation(_net(4, 4, 0), up, 0.0, 4.0, 9, twist=lambda s: 40.0 * s, taper=lambda s: 1.0 - 0.2 * s)
    moves = [_move(3, _translate(6, 0, 0), group=[3, 4], deform=d)]
    m, e_occ, e_lab = _replay_everywhere(occ, lab, moves)
    assert (m == 0).sum() > 10 and np.array_equal(m == 0, np.isin(e_lab, [3, 4]) & (e_occ > LEVEL))
    r, _, _, o, dd, x = _view(occ, lab, moves)
    moved = np.nonzero(r["move"] == 0)[0]
    assert moved.size
    trans = moves[0]["trans"]
    assert np.array_equal(r["point"][moved], DO.targets(moves[0], x[moved]))
    unit = DO.target_dirs(moves[0], x[moved], dd[moved])                    # the moved render's normalised direction
    v = r["dir"][moved]
    nrm = np.sqrt((v[:, 0] * v[:, 0] + v[:, 1] * v[:, 1]) + v[:, 2] * v[:, 2])
    assert np.array_equal((v / nrm[:, None]).astype(np.float32), unit)
    rigid = np.stack([(trans[a, 0] * dd[moved, 0].astype(np.float64) + trans[a, 1] * dd[moved, 1]) + trans[a, 2] * dd[moved, 2]
                      for a in range(3)], -1).astype(np.float32)
    assert not np.array_equal(v, rigid)                                        # the twist turned the direction


def test_a_vacate_after_a_take_keeps_the_taking_move():
    occ, lab = _scene()
    moves = [_move(3, _translate(6, 0, 0)), _move(3, _translate(0, 6, 0))]
    m, e_occ, e_lab = _replay_everywhere(occ, lab, moves)
    # the second move vacates what the first placed (its label is 3) and places the source's block again elsewhere
    assert (m[9:12, 3:6, 1:4] == 0).all() and (e_occ[9:12, 3:6, 1:4] == 0).all()
    assert (m[3:6, 9:12, 1:4] == 1).all() and (e_occ[3:6, 9:12, 1:4] > LEVEL).all()


def test_a_grid_that_is_not_the_edit_is_reported_at_its_hits():
    occ, lab = _scene()
    moves = [_move(3, _translate(6, 0, 0))]
    o, d = _rays()
    r = EV.edit_view(occ, lab, occ, lab, np.eye(4), EXT, o, d, 0.0, 100.0, moves, LEVEL)      # the source viewed as its edit
    assert r["mismatched"].any()
    c = r["cast"]
    assert (c["label"][r["mismatched"]] == 3).all()                                           # the block, which the move vacates
    e_occ, e_lab = _edited(occ, lab, moves)
    bad = e_occ.copy()
    bad[9, 4, 2] = np.nextafter(bad[9, 4, 2], np.float32(2))                                  # one bit of one moved point
    r2 = EV.edit_view(bad, e_lab, occ, lab, np.eye(4), EXT, o, d, 0.0, 100.0, moves, LEVEL)
    hits = r2["cast"]["voxel"] == (9 * DIM + 4) * DIM + 2
    assert hits.any() and np.array_equal(r2["mismatched"], hits)


def test_identity_move_gives_the_unedited_colour_inputs():
    occ, lab = _scene()
    moves = [_move(3, np.eye(4))]
    m, e_occ, e_lab = _replay_everywhere(occ, lab, moves)
    assert np.array_equal(e_occ.view(np.int32), occ.view(np.int32)) and np.array_equal(e_lab, lab)
    r, _, _, o, d, x = _view(occ, lab, moves)
    hit = r["cast"]["voxel"] >= 0
    assert np.array_equal(r["move"][hit] == 0, r["cast"]["label"][hit] == 3)
    assert np.array_equal(r["point"][hit], x[hit]) and np.array_equal(r["dir"][hit], d[hit])


# ---- grid_view's checks of moves= and source= -------------------------------------------------------------------------------

def _cpu_grid(dim=4):
    return torch.zeros((dim,) * 3), torch.zeros((dim,) * 3, dtype=torch.int16)


def _scene_moves(dim=4, T=np.eye(4), ext=(1.9, 7.0, 7.0), level=0.45, device="cpu"):
    d = _lib.RenderMoves()
    d.n_moves, d.dim = 1, dim
    d.transform[:] = np.asarray(T, dtype=np.float64).reshape(-1).tolist()
    d.extents[:] = list(ext)
    d.level, d.voxel = level, 0.1
    return OB.MovedScene(d, None, torch.device(device), (3,), np.zeros((1, 6), dtype=np.int64), (False,), level, 0.1)


@pytest.mark.parametrize("case, msg", [
    ("moves_only", "come together"), ("source_only", "come together"), ("not_moved_scene", "render_moves"),
    ("source_not_pair", "pair"), ("source_dim", "not the viewed grid"), ("source_dtype", "float32"),
    ("source_device", "source is on"), ("moves_device", "built on"), ("moves_dim", "dim"),
    ("moves_transform", "another grid"), ("moves_extents", "another grid"), ("moves_level", "level"),
])
def test_grid_view_checks_moves_and_source_before_device_work(case, msg):
    occ, lab = _cpu_grid()
    good_src = _cpu_grid()
    kw = dict(moves=_scene_moves(), source=good_src)
    if case == "moves_only":
        kw.pop("source")
    elif case == "source_only":
        kw.pop("moves")
    elif case == "not_moved_scene":
        kw["moves"] = [(3, np.eye(4))]
    elif case == "source_not_pair":
        kw["source"] = good_src[0]
    elif case == "source_dim":
        kw["source"] = _cpu_grid(5)
    elif case == "source_dtype":
        kw["source"] = (good_src[0].double(), good_src[1])
    elif case == "source_device":
        kw["source"] = tuple(t.to("meta") for t in good_src)
    elif case == "moves_device":
        kw["moves"] = _scene_moves(device="meta")
    elif case == "moves_dim":
        kw["moves"] = _scene_moves(dim=5)
    elif case == "moves_transform":
        T = np.eye(4)
        T[0, 3] = 0.5
        kw["moves"] = _scene_moves(T=T)
    elif case == "moves_extents":
        kw["moves"] = _scene_moves(ext=(2.0, 7.0, 7.0))
    elif case == "moves_level":
        kw["moves"] = _scene_moves(level=0.5)
    with pytest.raises(ValueError, match=msg):
        OB.grid_view(occ, lab, np.eye(4), 4, 4, np.eye(3), np.eye(4), 0.0, 1.0, **kw)


def test_grid_view_with_good_moves_and_source_still_needs_device_tensors():
    occ, lab = _cpu_grid()
    with pytest.raises(RuntimeError, match="CUDA"):
        OB.grid_view(occ, lab, np.eye(4), 4, 4, np.eye(3), np.eye(4), 0.0, 1.0, moves=_scene_moves(), source=_cpu_grid())
