"""CPU: the moving-pieces rule (DESIGN.md, "Moving pieces") in oracle/pieces_oracle.py: equal to the reference's exchanger without
pieces and with an all-ones region, the rule's cases on constructed raws with two pieces of one label, and the vote's sum."""
import os

import numpy as np
import pytest
import torch

from oracle import dmnerf_oracle as O
from oracle import pieces_oracle as P
from oracle import region_oracle as RO

INS = 3                  # labels 0 .. 3, 3 = "empty"
C = 4 + INS + 1
DIM = 4


def _words(labels):
    w = [0, 0, 0, 0]
    for k in labels:
        w[k >> 5] |= 1 << (k & 31)
    return w


def _region(mask, labels, outside_keep=False):
    """A region dict on a DIM^3 grid whose voxel map is the identity: point p is voxel rint(p)."""
    vmap = np.concatenate([np.eye(3), np.zeros((3, 1))], 1).astype(np.float32)
    return {"vmap": vmap, "bits": RO.pack(mask), "dim": DIM, "applies": _words(labels), "outside_keep": outside_keep}


def _piece_a(label=1):
    """Piece A = grid points with x index 0 or 1; the rest of the grid (x 2, 3) is piece B."""
    m = np.zeros((DIM, DIM, DIM), dtype=bool)
    m[:2] = True
    return _region(m, [label])


def _raw(labels, seed):
    """raw [N, S, C] whose arg-max label is `labels`, with distinct non-zero rgb / density values."""
    labels = np.asarray(labels)
    rng = np.random.default_rng(seed)
    raw = rng.uniform(0.5, 2.0, size=labels.shape + (C,)).astype(np.float32)
    raw[..., 4:] = -8.0
    np.put_along_axis(raw[..., 4:], labels[..., None], 8.0, -1)
    return torch.from_numpy(raw)


def _acc(labels):
    """A post-sigmoid accumulated instance map [N, INS + 1] whose arg-max over the first INS channels is `labels`."""
    acc = np.full((len(labels), INS + 1), 0.1, dtype=np.float32)
    acc[np.arange(len(labels)), labels] = 0.9
    return torch.from_numpy(acc)


def _rays(o, d):
    return torch.tensor(o, dtype=torch.float32), torch.tensor(d, dtype=torch.float32)


# rays along +x from x = 0 (first samples in A) or along -x from x = 3.2 (first samples in B); y = z = 1 inside the grid
ALONG, BACK = ([0.0, 1.0, 1.0], [1.0, 0.0, 0.0]), ([3.2, 1.0, 1.0], [-1.0, 0.0, 0.0])


def _scene():
    """Four rays of 4 samples, moved label 1 (the layout is spelled out per ray below)."""
    ori_o, ori_d = _rays(*zip(ALONG, ALONG, BACK, ALONG))
    ori_z = torch.tensor([[0.2, 1.0, 2.2, 3.0],      # ray 0: A A B bg, voted A: A moves away
                          [2.0, 2.5, 3.0, 3.2],      # ray 1: B B B bg, voted B: B stays (keep) or goes (drop)
                          [0.1, 0.5, 2.5, 3.0],      # ray 2: B B A A seen from x = 3.2: A behind B
                          [0.2, 1.0, 2.2, 3.0]])     # ray 3: background only
    ori_lab = [[1, 1, 1, 0], [1, 1, 1, 0], [1, 1, 1, 1], [0, 0, 0, 0]]
    tar_o, tar_d = _rays(*zip(ALONG, ALONG, ALONG, ALONG))
    tar_z = torch.tensor([[0.2, 1.0, 2.2, 3.0]] * 3 + [[0.3, 0.9, 2.5, 3.3]])
    tar_lab = [[0, 0, 0, 0]] * 3 + [[1, 1, 1, 0]]    # ray 3's target sees A (two samples) and B
    return {"ori_raw": _raw(ori_lab, 1), "tar_raw": _raw(tar_lab, 2), "ori_acc": _acc([1, 1, 1, 0]), "tar_acc": _acc([0, 0, 0, 1]),
            "ori_rays": (ori_o, ori_d), "ori_z": ori_z, "tar_rays": (tar_o, tar_d), "tar_z": tar_z,
            "ori_votes": np.array([[1, 0, 0, 1]], dtype=np.uint8), "tar_votes": np.array([1, 1, 1, 1], dtype=np.uint8)}


def _exchange(sc, rest_drop=False, region=None):
    pieces = {"regions": [_piece_a() if region is None else region], "rest_drop": [rest_drop], "ori_rays": sc["ori_rays"],
              "ori_z": sc["ori_z"], "tar_rays": [sc["tar_rays"]], "tar_zs": [sc["tar_z"]], "ori_votes": sc["ori_votes"],
              "tar_votes": [sc["tar_votes"]]}
    return P.exchanger_pieces(sc["ori_raw"], [sc["tar_raw"]], sc["ori_acc"], [sc["tar_acc"]], [1], pieces)


def test_the_regions_put_each_sample_where_the_scene_says():
    sc = _scene()
    inside = P.in_piece(_piece_a(), 1, *sc["ori_rays"], sc["ori_z"])
    assert inside.tolist() == [[True, True, False, False], [False, False, False, False], [False, False, True, True],
                               [True, True, False, False]]


def _golden():
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "manipulator.npz"))
    t = torch.from_numpy
    return (t(g["ex_ori_raw"]), [t(x) for x in g["ex_tar_raws"]], t(g["ex_acc_o"]), [t(x) for x in g["ex_acc_t"]],
            [int(v) for v in g["labels"]], t(g["ex_out_raw"]))


def test_without_pieces_and_with_an_all_ones_region_it_is_the_reference_exchanger():
    ori, tars, acc_o, acc_t, labels, want = _golden()
    ref = O.exchanger(ori, tars, acc_o, acc_t, labels)
    assert torch.equal(ref[0], want)
    got = P.exchanger_pieces(ori, tars, acc_o, acc_t, labels)
    for a, b in zip(got[2:], ref[2:]):
        assert torch.equal(a, b)
    assert torch.equal(got[0], ref[0])
    n, s, c = ori.shape
    rng = np.random.default_rng(5)
    rays = [_rays(rng.normal(size=(n, 3)) * 3, rng.normal(size=(n, 3))) for _ in range(len(labels) + 1)]
    zs = [torch.from_numpy(np.sort(rng.uniform(0, 9, size=(n, s)), -1).astype(np.float32)) for _ in rays]
    ones = {"vmap": RO.voxel_map(np.eye(3) * 0.1, np.zeros(3)), "bits": RO.pack(np.ones((8, 8, 8), dtype=bool)), "dim": 8,
            "applies": _words(range(c - 4)), "outside_keep": True}
    # the votes of an all-ones region are all 1 (nothing of the label is outside it)
    w = torch.from_numpy(rng.uniform(0, 0.2, size=(n, s)).astype(np.float32))
    votes = P.piece_vote(ori, zs[0], w, *rays[0], labels, [ones] * len(labels))
    assert votes.min() == 1
    for rest in (False, True):
        pieces = {"regions": [ones] * len(labels), "rest_drop": [rest] * len(labels), "ori_rays": rays[0], "ori_z": zs[0],
                  "tar_rays": rays[1:], "tar_zs": zs[1:], "ori_votes": votes, "tar_votes": [votes[0]] * len(labels)}
        got = P.exchanger_pieces(ori, tars, acc_o, acc_t, labels, pieces)
        for a, b in zip(got[:1] + got[2:], ref[:1] + ref[2:]):
            assert torch.equal(a, b)


def test_moving_piece_a_zeroes_its_old_samples_takes_its_target_and_keeps_or_drops_b():
    sc = _scene()
    o, t = sc["ori_raw"], sc["tar_raw"]
    zero = o * 0
    for rest_drop in (False, True):
        out, _, lab, tlab = _exchange(sc, rest_drop)
        # ray 0 (voted A): A's samples moved away; its other samples are filled from the target (the reference's filling)
        assert torch.equal(out[0, :2], zero[0, :2]) and torch.equal(out[0, 2:], t[0, 2:])
        # ray 1 (voted B): B stays with `keep`, vanishes with `drop`; its background sample stays
        assert torch.equal(out[1, :3], zero[1, :3] if rest_drop else o[1, :3]) and torch.equal(out[1, 3], o[1, 3])
        # ray 3: the target's two samples of A are taken, its sample of B is not
        assert torch.equal(out[3, :2], t[3, :2]) and torch.equal(out[3, 2:], o[3, 2:])
        assert tlab[3].tolist() == [1, 1, 1, 0]


def test_a_behind_b_follows_the_occlusion_fix():
    sc = _scene()
    o = sc["ori_raw"]
    out, _, lab, _ = _exchange(sc)
    # ray 2 is voted B: A's samples behind B take the ray's label, whose vote says "not the piece", and stay
    assert torch.equal(out[2], o[2])
    assert lab[2].tolist() == [1, 1, 1, 1]
    # with `drop`, every sample labelled 1 on that ray is the rest of the label
    out, _, _, _ = _exchange(sc, rest_drop=True)
    assert torch.equal(out[2], o[2] * 0)
    # the reference's exchanger moves the whole label: the ray empties
    ref = O.exchanger(o, [sc["tar_raw"]], sc["ori_acc"], [sc["tar_acc"]], [1])
    assert torch.equal(ref[0][2], o[2] * 0)


def test_a_vote_tie_counts_as_moving():
    n, s = 3, 4
    lab = [[1, 1, 0, 0], [1, 1, 0, 0], [0, 0, 0, 0]]
    raw = _raw(lab, 3)
    ro, rd = _rays([ALONG[0]] * n, [ALONG[1]] * n)
    z = torch.tensor([[0.5, 2.5, 3.0, 3.1], [0.5, 2.5, 3.0, 3.1], [0.5, 2.5, 3.0, 3.1]])
    w = torch.tensor([[0.25, 0.25, 0.1, 0.1], [0.25, 0.5, 0.1, 0.1], [0.3, 0.3, 0.2, 0.1]])
    # ray 0: in = out = 0.25 (tie), ray 1: in < out, ray 2: no sample of the label: 0 = 0
    assert P.piece_vote(raw, z, w, ro, rd, [1], [_piece_a()]).tolist() == [[1, 0, 1]]
    # without a region every vote is 1
    assert P.piece_vote(raw, z, w, ro, rd, [1], [None]).tolist() == [[1, 1, 1]]
    # a tied ray's accumulated label is the moving piece: its samples of the label outside the piece are filled
    sc = _scene()
    sc["ori_votes"] = np.array([[1, 1, 1, 1]], dtype=np.uint8)
    out, _, _, _ = _exchange(sc)
    assert torch.equal(out[1, :3], sc["tar_raw"][1, :3])


def test_with_two_moves_a_label_copied_from_acc_is_judged_by_its_vote():
    """Move 1 (label 1, piece A) relabels an A sample on a ray that accumulates label 2; move 2 (label 2, a region of no points)
    then moves it when the ray's vote for move 2 is 1, although its point is not in move 2's piece, and leaves it when it is 0."""
    lab = [[1, 0, 0, 0]]
    ori = _raw(lab, 4)
    tars = [_raw([[0, 0, 0, 0]], 5), _raw([[0, 0, 0, 0]], 6)]
    ro, rd = _rays([ALONG[0]], [ALONG[1]])
    z = torch.tensor([[0.2, 2.2, 3.0, 3.1]])
    none = _region(np.zeros((DIM, DIM, DIM), dtype=bool), [2])
    assert not P.in_piece(none, 2, ro, rd, z).any()
    for vote2, moved in ((1, True), (0, False)):
        pieces = {"regions": [_piece_a(), none], "rest_drop": [False, False], "ori_rays": (ro, rd), "ori_z": z,
                  "tar_rays": [(ro, rd)] * 2, "tar_zs": [z] * 2, "ori_votes": np.array([[1], [vote2]], dtype=np.uint8),
                  "tar_votes": [np.array([1], dtype=np.uint8)] * 2}
        out, _, lab_out, _ = P.exchanger_pieces(ori, tars, _acc([2]), [_acc([0]), _acc([0])], [1, 2], pieces)
        assert lab_out[0, 0] == 2
        assert torch.equal(out[0, 0], ori[0, 0] * 0 if moved else ori[0, 0]), vote2
        # the ray's other samples are filled from target 2 when the ray is the moving piece of move 2
        assert torch.equal(out[0, 1:], tars[1][0, 1:] if moved else ori[0, 1:])


def test_piece_vote_against_a_float64_sum():
    rng = np.random.default_rng(11)
    n, s, dim = 300, 96, 16
    labels = rng.integers(0, INS + 1, size=(n, s))
    raw = _raw(labels, 7)
    mask = rng.random((dim, dim, dim)) < 0.5
    reg = {"vmap": RO.voxel_map(np.eye(3) * (2.0 / (dim - 1)), -np.ones(3)), "bits": RO.pack(mask), "dim": dim,
           "applies": _words([1, 2]), "outside_keep": False}
    ro = rng.uniform(-1.5, 1.5, size=(n, 3)).astype(np.float32)
    rd = rng.normal(size=(n, 3)).astype(np.float32) * 0.3
    z = np.sort(rng.uniform(0, 4, size=(n, s)), -1).astype(np.float32)
    w = rng.uniform(0, 0.05, size=(n, s)).astype(np.float32)
    got = P.piece_vote(raw, torch.from_numpy(z), torch.from_numpy(w), torch.from_numpy(ro), torch.from_numpy(rd), [1, 2], [reg, reg])
    for i, mv in enumerate((1, 2)):
        inside = P.in_piece(reg, mv, ro, rd, z)
        lab = labels == mv
        d_in = np.where(lab & inside, w.astype(np.float64), 0).sum(1)
        d_out = np.where(lab & ~inside, w.astype(np.float64), 0).sum(1)
        clear = np.abs(d_in - d_out) > 1e-5 * np.maximum(d_in + d_out, 1e-30)        # away from ties
        assert clear.mean() > 0.9
        assert np.array_equal(got[i][clear], (d_in >= d_out)[clear].astype(np.uint8))
        assert np.array_equal(got[i][(d_in + d_out) == 0], np.ones(int(((d_in + d_out) == 0).sum()), dtype=np.uint8))


def test_a_moved_label_outside_the_regions_labels_is_refused():
    sc = _scene()
    with pytest.raises(ValueError):
        _exchange(sc, region=_piece_a(label=2))
