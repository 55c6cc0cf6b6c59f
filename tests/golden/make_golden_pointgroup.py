"""Golden vectors for PointGroup's segmentation network, produced by EXECUTING THE REFERENCE's own PointGroup model
(PointGroup/model/pointgroup/pointgroup.py) inside its own PointGroupPredictor.predict (predicter.py:232-338), with
the real sklearn MeanShift and scipy cKDTree.

Run in the authoring container only (needs the reference checkout at /root/reference):

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_pointgroup.py

Stand-ins for what does not build here, each computing in float64:
  * spconv: SparseConvTensor, SparseSequential (spconv 1.x's forward: sparse modules take the tensor, the others its
    features), SparseModule, SubMConv3d, SparseConv3d and SparseInverseConv3d with spconv 1.x parameter shapes
    (k, k, k, Cin, Cout) + bias, computing through oracle/spconv_ref (neighbours by lookup in the tensor's own row
    order; an inverse conv reuses the pairs its indice_key's SparseConv3d stored);
  * pointgroup_ops.voxelization_idx / voxelization: oracle/pointgroup_ref's restatement of mode 4;
  * open3d's voxel_down_sample: oracle.cloud_ref.voxel_down_sample.
The reference's code decides the module tree, the state_dict keys, the concatenation order, where the residuals go
and the host front.  The model runs in float64 (model.double()); its pt_offsets are rounded to float32 once, where
predict reads them.  The weights are oracle.pointgroup_ref.synthetic_state_dict(key shapes, SEED), saved as a
checkpoint with 'module.' prefixes and loaded by the reference's load_model (strict).

pointgroup.npz holds key_shapes (JSON [[key, shape]] of the reference model's state_dict without num_batches_tracked),
seed, m, block_reps, and per class (prefix hnm_, nut_, screw_): cloud_xyz, cloud_normal (the predict input, float32, a
make_pile scene thinned so that no two points share a 2 mm voxel),
xyz_original_all, locs (N,3) int64, spatial_shape, sites (V,3) in the reference's first-seen order, p2v (N,), vfeats
(V,6) float32, offsets64 (N,3) (the reference model in float64) with bound (N,3) (oracle/pointgroup_ref's propagated
bound), labels_all and xyz_shifted (the reference's results), scene_seed (the make_pile seed), and stable_seeds: the
seeds of the +-1e-6 m offset perturbations under which labels_all did not change (all of them: a scene whose labels
move is skipped for the next seed).
"""
import json
import os
import sys
import tempfile
import types
import importlib.util

import numpy as np
import torch
import torch.nn as nn

sys.dont_write_bytecode = True
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", ".."))
REF = "/root/reference"
sys.path.insert(0, REF)

from oracle import cloud_ref, spconv_ref                # noqa: E402
from oracle import pointgroup_ref as PR                  # noqa: E402
from catgrasp_b200 import synthetic                      # noqa: E402

SEED = 7
STABLE_SEEDS = (1, 2, 3)


class _Any:
    def __init__(self, *a, **k):
        pass

    def __call__(self, *a, **k):
        return _Any()

    def __getattr__(self, n):
        return _Any()


class _Stub(types.ModuleType):
    __all__ = []
    __path__ = []

    def __getattr__(self, name):
        if name.startswith("__"):
            raise AttributeError(name)
        full = self.__name__ + "." + name
        if full in sys.modules:
            return sys.modules[full]
        return type(name, (_Any,), {})


# ---------------------------------------------------------------- the spconv stand-in
def _subm_nbr(ind):
    """SubM k3 table in the rows' own order: nbr[r][k] = the row at ind[r] + (kx-1, ky-1, kz-1)."""
    keys = spconv_ref.pack(ind)
    order = np.argsort(keys)
    sk = keys[order]
    nbr = np.full((len(ind), 27), -1, dtype=np.int64)
    for k in range(27):
        q = ind + np.array([k // 9 - 1, k // 3 % 3 - 1, k % 3 - 1])
        ok = (q >= 0).all(1)
        qk = spconv_ref.pack(np.where(ok[:, None], q, 0))
        pos = np.minimum(np.searchsorted(sk, qk), len(sk) - 1)
        hit = ok & (sk[pos] == qk)
        nbr[hit, k] = order[pos[hit]]
    return nbr


class SparseConvTensor:
    def __init__(self, features, indices, spatial_shape, batch_size, grid=None):
        self.features, self.indices = features, indices
        self.spatial_shape, self.batch_size = [int(s) for s in spatial_shape], batch_size
        self.indice_dict = {}

    @property
    def sparity(self):
        return 1.0

    def sites(self):
        return np.asarray(self.indices)[:, 1:].astype(np.int64)


class SparseModule(nn.Module):
    pass


class SparseSequential(nn.Sequential):
    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self._sparity_dict = {}

    def forward(self, input):                      # spconv 1.x modules.py SparseSequential.forward
        for k, module in self._modules.items():
            if isinstance(module, SparseModule):
                input = module(input)
            elif isinstance(input, SparseConvTensor):
                if input.indices.shape[0] != 0:
                    input.features = module(input.features)
            else:
                input = module(input)
        return input


class _Conv(SparseModule):
    def __init__(self, in_channels, out_channels, kernel_size=3, stride=1, padding=0, bias=True, indice_key=None):
        super().__init__()
        self.k, self.indice_key = int(kernel_size), indice_key
        self.weight = nn.Parameter(torch.zeros((self.k,) * 3 + (in_channels, out_channels)))
        self.bias = nn.Parameter(torch.zeros(out_channels)) if bias else None

    def _run(self, x, nbr):
        W = self.weight.detach().double().numpy().reshape(-1, self.weight.shape[-2], self.weight.shape[-1])
        b = None if self.bias is None else self.bias.detach().double().numpy()
        y, _ = spconv_ref.conv(x.detach().double().numpy(), nbr, W, bias=b)
        return torch.from_numpy(y)

    def _out(self, t, feats, indices, shape):
        o = SparseConvTensor(feats, indices, shape, t.batch_size)
        o.indice_dict = t.indice_dict
        return o


class SubMConv3d(_Conv):
    def forward(self, t):
        nbr = None if self.k == 1 else _subm_nbr(t.sites())
        return self._out(t, self._run(t.features, nbr), t.indices, t.spatial_shape)


class SparseConv3d(_Conv):
    def forward(self, t):
        assert self.k == 2
        cvox, _, dn, up, cshape = spconv_ref.down(t.sites(), t.spatial_shape)
        t.indice_dict[self.indice_key] = (t.indices, t.spatial_shape, up)
        cind = np.concatenate([np.zeros((len(cvox), 1), np.int64), cvox.astype(np.int64)], 1)
        return self._out(t, self._run(t.features, dn), torch.from_numpy(cind), cshape)


class SparseInverseConv3d(_Conv):
    def __init__(self, in_channels, out_channels, kernel_size, indice_key, bias=True):
        super().__init__(in_channels, out_channels, kernel_size, bias=bias, indice_key=indice_key)

    def forward(self, t):
        ind, shape, up = t.indice_dict[self.indice_key]
        return self._out(t, self._run(t.features, up), ind, shape)


_spconv = types.ModuleType("spconv")
for _c in (SparseConvTensor, SparseSequential, SparseModule, SubMConv3d, SparseConv3d, SparseInverseConv3d):
    setattr(_spconv, _c.__name__, _c)
_spconv.modules = types.ModuleType("spconv.modules")
_spconv.modules.SparseModule = SparseModule
sys.modules["spconv"], sys.modules["spconv.modules"] = _spconv, _spconv.modules


# ---------------------------------------------------------------- pointgroup_ops stand-in, other absent modules
def _voxelization_idx(locs, batch_size, mode):
    assert mode == 4
    vl, p2v, v2p = PR.voxelization_idx(locs.numpy())
    return torch.from_numpy(vl), torch.from_numpy(p2v), torch.from_numpy(v2p)


def _voxelization(feats, v2p, mode):
    assert mode == 4
    return torch.from_numpy(PR.voxelization(feats.numpy(), v2p.numpy()))


_ABSENT = ["open3d", "trimesh", "transformations", "autolab_core", "matplotlib", "matplotlib.pyplot", "pybullet",
           "dexnet", "dexnet.grasping", "dexnet.grasping.grasp", "dexnet.grasping.gripper",
           "dexnet.grasping.grasp_sampler",
           "PointGroup", "PointGroup.data", "PointGroup.data.dataset_seg", "PointGroup.model",
           "PointGroup.model.pointgroup", "PointGroup.lib", "PointGroup.lib.pointgroup_ops",
           "PointGroup.lib.pointgroup_ops.functions", "PointGroup.lib.pointgroup_ops.functions.pointgroup_ops",
           "PointGroup.util", "PointGroup.util.config",
           "lib", "lib.pointgroup_ops", "lib.pointgroup_ops.functions", "lib.pointgroup_ops.functions.pointgroup_ops"]
for _m in _ABSENT:
    sys.modules[_m] = _Stub(_m)
for _m in ("PointGroup.lib.pointgroup_ops.functions.pointgroup_ops", "lib.pointgroup_ops.functions.pointgroup_ops"):
    sys.modules[_m].voxelization_idx = _voxelization_idx
    sys.modules[_m].voxelization = _voxelization
sys.modules["lib.pointgroup_ops.functions"].pointgroup_ops = sys.modules["lib.pointgroup_ops.functions.pointgroup_ops"]
torch.Tensor.cuda = lambda self, *a, **k: self


class _PointCloud:
    """open3d.geometry.PointCloud with the one method predict uses, voxel_down_sample = the oracle's."""

    def __init__(self):
        self.points = np.zeros((0, 3))

    def voxel_down_sample(self, voxel_size):
        out = _PointCloud()
        out.points = cloud_ref.voxel_down_sample(np.asarray(self.points, np.float64), voxel_size)[0]
        return out


o3d = sys.modules["open3d"]
o3d.geometry = types.SimpleNamespace(PointCloud=_PointCloud)
o3d.utility = types.SimpleNamespace(Vector3dVector=lambda a: np.asarray(a, np.float64).copy())


def _load(name, path):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    sys.modules[name] = mod
    spec.loader.exec_module(mod)
    return mod


sys.path.insert(0, os.path.join(REF, "PointGroup"))
_cfgmod = _load("PointGroup.util.config", os.path.join(REF, "PointGroup", "util", "config.py"))
_pgmod = _load("PointGroup.model.pointgroup.pointgroup",
               os.path.join(REF, "PointGroup", "model", "pointgroup", "pointgroup.py"))
import predicter as ref_predicter                        # noqa: E402  the reference itself


class _Net:
    """The reference model in float64; predict reads its pt_offsets rounded to float32 once.  ``perturb`` adds a
    seeded uniform +-1e-6 m to them."""

    def __init__(self, model, perturb=None):
        self.model, self.prepare_epochs, self.perturb, self.seen = model, model.prepare_epochs, perturb, None

    def __call__(self, input_, p2v_map, coords_float, *a, **k):
        self.seen = {"sites": input_.indices[:, 1:].numpy().astype(np.int32).copy(),
                     "vfeats": input_.features.numpy().copy(), "p2v": p2v_map.numpy().astype(np.int32).copy(),
                     "spatial_shape": np.asarray(input_.spatial_shape, np.int64)}
        with torch.no_grad():
            off = self.model(input_, p2v_map, coords_float.double(), *a, **k)["pt_offsets"].numpy()
        self.seen["offsets64"] = off.copy()
        off32 = off.astype(np.float32)
        if self.perturb is not None:
            off32 = (off32 + np.random.RandomState(self.perturb).uniform(-1e-6, 1e-6, off.shape)).astype(np.float32)
        return {"pt_offsets": torch.from_numpy(off32)}


def _config():
    with open(os.path.join(REF, "PointGroup", "config", "config_pointgroup.yaml")) as f:
        import yaml
        return _cfgmod.key_to_attr(types.SimpleNamespace(), yaml.safe_load(f))


def _model(cfg, tmp):
    model = _pgmod.PointGroup(cfg)
    key_shapes = [(k, tuple(v.shape)) for k, v in model.state_dict().items() if not k.endswith("num_batches_tracked")]
    sd = PR.synthetic_state_dict(key_shapes, SEED)
    ck = {"state_dict": {"module." + k: torch.from_numpy(v) for k, v in sd.items()}}
    path = os.path.join(tmp, "best_val.pth.tar")
    torch.save(ck, path)
    ref_predicter.load_model(model, ckpt_dir=path)
    for k, v in sd.items():                              # strict load took every value
        assert np.array_equal(model.state_dict()[k].numpy(), v), k
    return model.double().eval(), key_shapes, sd


def _predictor(class_name, cfg, net):
    p = ref_predicter.PointGroupPredictor.__new__(ref_predicter.PointGroupPredictor)
    p.class_name, p.n_slice_per_side, p.cfg_pg = class_name, 1, cfg
    p.cfg = {"downsample_size": 0.0005}                                   # config_pointgroup.yaml:13
    p.dataset = types.SimpleNamespace(scale=cfg.scale, full_scale=cfg.full_scale, mode=cfg.mode)
    p.model = net
    return p


THIN = 0.002 * np.sqrt(3.0) * 1.01


def thin(xyz, spacing):
    """Greedy subset with no two points within `spacing` (ascending index order)."""
    from scipy.spatial import cKDTree
    nbrs = cKDTree(xyz).query_ball_point(xyz, spacing)
    keep = np.ones(len(xyz), bool)
    for i in range(len(xyz)):
        if keep[i]:
            keep[[j for j in nbrs[i] if j > i]] = False
    return np.nonzero(keep)[0]


def run(class_name, cfg, model, sd, n_points, n_objects, seed):
    scene = synthetic.make_pile(n_points, n_objects=n_objects, seed=seed)
    # no two points share a 2 mm voxel (so none shares a 0.5 mm one either): a voxel of two points has its mean
    # midway between them, and cKDTree answers that tie with whichever point its traversal meets, which no other
    # implementation can reproduce
    sel = thin(scene["cloud_xyz"], THIN)
    data = {"cloud_xyz": scene["cloud_xyz"][sel].astype(np.float32),
            "cloud_normal": scene["cloud_normal"][sel].astype(np.float32), "cloud_rgb": np.zeros((len(sel), 3), np.uint8)}
    net = _Net(model)
    p = _predictor(class_name, cfg, net)
    labels_all = np.asarray(p.predict({k: v.copy() for k, v in data.items()}), np.int64)
    s = net.seen
    xo, locs, feats, shape = PR.host_front(data["cloud_xyz"], data["cloud_normal"])
    assert np.array_equal(shape, s["spatial_shape"])
    off, bound, _, _ = PR.forward(sd, cfg.m, cfg.block_reps, s["sites"], shape, s["vfeats"], s["p2v"])
    scale = np.abs(s["offsets64"]).max()
    agree = np.abs(off - s["offsets64"]).max() / scale
    assert agree < 1e-10, agree                                          # the oracle's wiring == the reference's
    stable = []
    for ps in STABLE_SEEDS:
        q = _predictor(class_name, cfg, _Net(model, perturb=ps))
        if np.array_equal(np.asarray(q.predict({k: v.copy() for k, v in data.items()}), np.int64), labels_all):
            stable.append(ps)
    return {"cloud_xyz": data["cloud_xyz"], "cloud_normal": data["cloud_normal"], "xyz_original_all": xo,
            "locs": locs, "spatial_shape": shape, "sites": s["sites"], "p2v": s["p2v"], "vfeats": s["vfeats"],
            "offsets64": s["offsets64"], "bound": bound, "labels_all": labels_all,
            "xyz_shifted": np.asarray(p.xyz_shifted, np.float32), "stable_seeds": np.asarray(stable, np.int64)}, agree


def main():
    cfg = _config()
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        model, key_shapes, sd = _model(cfg, tmp)
    out["key_shapes"] = np.array(json.dumps([[k, list(s)] for k, s in key_shapes]))
    out["seed"], out["m"], out["block_reps"] = np.int64(SEED), np.int64(cfg.m), np.int64(cfg.block_reps)
    for class_name, n, k, seed in (("hnm", 30000, 10, 51), ("nut", 40000, 16, 52), ("screw", 30000, 10, 53)):
        while True:                  # the first scene from `seed` on whose labels survive every perturbation
            r, agree = run(class_name, cfg, model, sd, n, k, seed)
            if len(r["stable_seeds"]) == len(STABLE_SEEDS):
                break
            print(class_name, "scene seed", seed, "labels moved under", sorted(set(STABLE_SEEDS) - set(r["stable_seeds"])))
            seed += 100
        r["scene_seed"] = np.int64(seed)
        for key, v in r.items():
            out[f"{class_name}_{key}"] = v
        print(class_name, "scene seed", seed, "points", len(r["xyz_original_all"]), "sites", len(r["sites"]),
              "clusters", len(np.unique(r["labels_all"])), "oracle/reference rel diff", f"{agree:.1e}",
              "max |offset|", f"{np.abs(r['offsets64']).max():.2e}", "stable under seeds", r["stable_seeds"].tolist())
    np.savez_compressed(os.path.join(HERE, "pointgroup.npz"), **out)


if __name__ == "__main__":
    main()
