"""PointGroup without a GPU: oracle/pointgroup_ref.py against tests/golden/pointgroup.npz (the reference's own model and
predict, see make_golden_pointgroup.py), the checkpoint loader of weights.py and PointGroupPredictor's config checks.
"""
import json
import os

import numpy as np
import pytest
import yaml

from catgrasp_b200 import weights
from catgrasp_b200.predicter import PointGroupPredictor, flatten_config, slice_keep_mask
from oracle import pointgroup_ref as PR

G = np.load(os.path.join(os.path.dirname(__file__), "golden", "pointgroup.npz"))
CLASSES = ("hnm", "nut", "screw")
KEY_SHAPES = [(k, tuple(s)) for k, s in json.loads(str(G["key_shapes"]))]
M, REPS = int(G["m"]), int(G["block_reps"])


def golden_state_dict():
    return PR.synthetic_state_dict(KEY_SHAPES, int(G["seed"]))


@pytest.mark.parametrize("cls", CLASSES)
def test_host_front_matches_golden(cls):
    xo, locs, feats, shape = PR.host_front(G[f"{cls}_cloud_xyz"], G[f"{cls}_cloud_normal"])
    assert np.array_equal(xo, G[f"{cls}_xyz_original_all"])
    assert np.array_equal(locs, G[f"{cls}_locs"]) and np.array_equal(shape, G[f"{cls}_spatial_shape"])
    locs4 = np.concatenate([np.zeros((len(locs), 1), np.int64), locs], 1)
    vl, p2v, v2p = PR.voxelization_idx(locs4)
    assert np.array_equal(vl[:, 1:], G[f"{cls}_sites"]) and np.array_equal(p2v, G[f"{cls}_p2v"])
    vf = PR.voxelization(feats, v2p)
    assert np.array_equal(vf.view(np.uint32), G[f"{cls}_vfeats"].view(np.uint32))


@pytest.mark.parametrize("cls", CLASSES)
def test_oracle_forward_matches_golden(cls):
    off, bound, _, _ = PR.forward(golden_state_dict(), M, REPS, G[f"{cls}_sites"], G[f"{cls}_spatial_shape"],
                                  G[f"{cls}_vfeats"], G[f"{cls}_p2v"])
    ref = G[f"{cls}_offsets64"]
    assert (np.abs(off - ref) <= G[f"{cls}_bound"]).all()
    assert np.abs(off - ref).max() <= 1e-9 * np.abs(ref).max()
    assert np.array_equal(bound, G[f"{cls}_bound"])


def test_keep_mask_drops_float32_xmax():
    # in float32, xmin + (xmax - xmin) rounds below xmax here, so the reference drops the point at xmax
    xmin, xmax = np.float32(-0.07290356), np.float32(0.19376823)
    assert xmin + (xmax - xmin) < xmax
    xyz = np.array([[xmin, 0, 0.7], [0.05, 0.1, 0.7], [xmax, 0.2, 0.7]], np.float32)
    assert slice_keep_mask(xyz).tolist() == [True, True, False]
    assert slice_keep_mask(xyz.astype(np.float64)).tolist() == [True, True, True]
    nrm = np.tile(np.float32([0, 0, 1]), (3, 1))
    xo, _, _, _ = PR.host_front(xyz, nrm, downsample_size=0.0005)
    assert len(xo) == 2 and xmax not in xo[:, 0]


def test_keys_match_reference_model():
    assert list(weights.pointgroup_keys(M, REPS).items()) == KEY_SHAPES
    # the widest tail input at m = 32 is 12 m = 384 channels (level 6's first tail block)
    k32 = weights.pointgroup_keys(32, 2)
    assert k32["unet." + "u." * 5 + "blocks_tail.block0.conv_branch.2.weight"] == (3, 3, 3, 384, 192)


def test_loader_strict_and_strips_module():
    sd = golden_state_dict()
    ck = {"state_dict": {"module." + k: v for k, v in sd.items()}}
    packed = weights.pack_pointgroup(ck, M, REPS)
    assert len(packed["levels"]) == 7 and packed["head"]["W1"].shape == (M, M)
    assert packed["levels"][0]["tail"][0]["Wi"].shape == (1, 2 * M, M)
    assert packed["levels"][6].get("down") is None
    missing = dict(sd)
    del missing["unet.u.conv.0.running_var"]
    with pytest.raises(RuntimeError, match="unet.u.conv.0.running_var"):
        weights.pack_pointgroup(missing, M, REPS)
    extra = dict(sd, **{"unet.extra.weight": np.zeros(3, np.float32)})
    with pytest.raises(RuntimeError, match="unet.extra.weight"):
        weights.pack_pointgroup(extra, M, REPS)
    bad = dict(sd, **{"offset.0.weight": np.zeros((M, M + 1), np.float32)})
    with pytest.raises(ValueError, match="offset.0.weight"):
        weights.pack_pointgroup(bad, M, REPS)
    no_score = {k: v for k, v in sd.items() if not k.startswith("score_")}
    with pytest.raises(RuntimeError, match="score_"):
        weights.pack_pointgroup(no_score, M, REPS)


def test_bn_packing_is_float64_then_narrowed():
    sd = golden_state_dict()
    s, t = weights.pack_pointgroup(sd, M, REPS)["levels"][0]["blocks"][0]["bn1"]
    p = "unet.blocks.block0.conv_branch.0"
    g, b, mu, var = (sd[p + x].astype(np.float64) for x in (".weight", ".bias", ".running_mean", ".running_var"))
    s64 = g / np.sqrt(var + 1e-5)
    assert s.dtype == np.float32 and np.array_equal(s, s64.astype(np.float32))
    assert np.array_equal(t, (b - mu * s64).astype(np.float32))


SHIPPED = {"GENERAL": {"input_channel": 3, "scale": 500, "full_scale": [128, 999999], "mode": 4},
           "STRUCTURE": {"m": 16, "block_residual": True, "block_reps": 2, "use_coords": True},
           "GROUP": {"prepare_epochs": 999999}, "downsample_size": 0.0005, "class_name": "nut"}


def test_flatten_config():
    flat = flatten_config(SHIPPED)
    assert flat["m"] == 16 and flat["mode"] == 4 and flat["full_scale"] == [128, 999999]
    assert flat["downsample_size"] == 0.0005 and "STRUCTURE" not in flat
    assert flatten_config({"A": {"x": 1}, "B": {"x": 2}})["x"] == 2     # setattr order: the later section wins


@pytest.mark.parametrize("section,key,value", [("GENERAL", "mode", 3), ("STRUCTURE", "use_coords", False),
                                               ("STRUCTURE", "block_residual", False),
                                               ("GENERAL", "input_channel", 6), ("STRUCTURE", "block_reps", 3)])
def test_unsupported_structure_raises(tmp_path, section, key, value):
    cfg = json.loads(json.dumps(SHIPPED))
    cfg[section][key] = value
    (tmp_path / "config_pointgroup.yaml").write_text(yaml.safe_dump(cfg))
    with pytest.raises(NotImplementedError, match=key):
        PointGroupPredictor("nut", artifact_dir=str(tmp_path))


def test_n_slice_per_side_other_than_one_raises():
    p = PointGroupPredictor.__new__(PointGroupPredictor)
    p.cfg_pg, p.n_slice_per_side = flatten_config(SHIPPED), 2
    with pytest.raises(NotImplementedError, match="n_slice_per_side"):
        p._check_structure()
