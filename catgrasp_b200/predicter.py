"""GraspPredicter / NunocsPredicter with the reference's call surface (predicter.py:39-203).

Host side (numpy, identical RNG consumption to the reference):
  * z >= 0.1 mask and the per-candidate ``np.random.choice`` subset (dataset_grasp.py:64,72-73;
    dataset_nunocs.py:40-44) -- only the *indices* are drawn on the host;
  * NUNOCS min/max-extent normalisation (augmentations.py:70-75);
  * the 9-DoF RANSAC (aligning.py:83-119) stays a host stage (SURVEY.md 8f F1).
Device side (libcatgrasp_b200.so): per-candidate rigid transform + normalisation + PointNet forward
+ softmax / argmax post-processing.
"""
import copy
import os
import pickle

import numpy as np
import yaml

from .net import PointNetCls, PointNetSeg
from .weights import load_checkpoint

_CODE_DIR = os.environ.get("CATGRASP_CODE_DIR", os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def to_homo(pts):
    """Utils.py:396-402."""
    assert len(pts.shape) == 2, f"pts.shape: {pts.shape}"
    return np.concatenate((pts, np.ones((pts.shape[0], 1))), axis=-1)


def _load_artifacts(artifact_dir, cfg_name):
    with open(f"{artifact_dir}/{cfg_name}", "r") as ff:
        cfg = yaml.safe_load(ff)
    normalizer_dir = f"{artifact_dir}/normalizer.pkl"
    if os.path.exists(normalizer_dir):          # predicter.py:53-58 / :122-126
        with open(normalizer_dir, "rb") as ff:
            tmp = pickle.load(ff)
        cfg["mean"] = np.asarray(tmp["mean"], dtype=np.float64)
        cfg["std"] = np.asarray(tmp["std"], dtype=np.float64)
    return cfg


def draw_subsample_ids_numpy(M, n_pts, count):
    """The draw exactly as the reference makes it: one np.random.choice per candidate (kept as the pin for the C path)."""
    replace = M < n_pts
    pop = np.arange(M)
    out = np.empty((count, n_pts), dtype=np.int32)
    for i in range(count):
        out[i] = np.random.choice(pop, size=(n_pts), replace=replace)
    return out


class _LegacyDraw:
    """Bit-identical continuation of numpy's GLOBAL legacy generator in C (cg_host_legacy_choice): take the MT19937
    state once, draw any number of candidates (possibly in chunks, from a worker thread), put the advanced state back."""

    def __init__(self):
        import ctypes as C
        from . import _lib
        self._C, self._lib = C, _lib.load()
        st = np.random.get_state()
        assert st[0] == "MT19937"
        self._rest = (st[3], st[4])
        self.key = np.ascontiguousarray(st[1], dtype=np.uint32).copy()
        self.pos = C.c_int32(int(st[2]))

    def draw(self, M, n_pts, count, out=None, nthreads=0):
        if out is None:
            out = np.empty((count, n_pts), dtype=np.int32)
        rc = self._lib.cg_host_legacy_choice(self.key, self._C.byref(self.pos), M, n_pts, count, out, nthreads)
        if rc != 0:
            raise ValueError(f"cg_host_legacy_choice({M}, {n_pts}, {count}) failed with {rc}")
        return out

    def skip(self, M, n_pts, count):
        rc = self._lib.cg_host_legacy_skip(self.key, self._C.byref(self.pos), M, n_pts, count)
        if rc != 0:
            raise ValueError(f"cg_host_legacy_skip({M}, {n_pts}, {count}) failed with {rc}")

    def commit(self):
        np.random.set_state(("MT19937", self.key, int(self.pos.value), self._rest[0], self._rest[1]))


def draw_subsample_ids(M, n_pts, count=None):
    """The reference's per-sample index draw (dataset_grasp.py:72-73, dataset_nunocs.py:43-44):
    ``np.random.choice(np.arange(M), size=n_pts, replace=M < n_pts)`` from the GLOBAL numpy RNG,
    once per candidate, in candidate order.  With ``count`` the draws run in C on numpy's own MT19937 state
    (same indices, same state afterwards -- tests/test_abi_and_host.py compares with numpy itself)."""
    if count is None:
        return np.random.choice(np.arange(M), size=(n_pts), replace=M < n_pts).astype(np.int32)
    d = _LegacyDraw()
    out = d.draw(M, n_pts, count)
    d.commit()
    return out


class GraspPredicter:
    """predicter.py:39-94."""

    class_name_to_artifact_id = {"nut": 47, "hnm": 51, "screw": 50}

    ENGINE_TOL = 2e-5   # load-time gate of the fast engine: max |dprob| against the near-fp32 engine on a probe batch

    def __init__(self, class_name, artifact_dir=None, device=None, engine="auto"):
        artifact_id = self.class_name_to_artifact_id[class_name]
        if artifact_dir is None:
            artifact_dir = f"{_CODE_DIR}/artifacts/artifacts-{artifact_id}"
        print("GraspPredicter artifact_dir", artifact_dir)
        self.class_name = class_name
        self.cfg = _load_artifacts(artifact_dir, "config_grasp.yml")
        n_out = len(self.cfg["classes"]) - 1
        assert self.cfg["input_channel"] == 6, "the H100 path implements the shipped 6-channel input"
        sd = load_checkpoint(f"{artifact_dir}/best_val.pth.tar")
        print("Load ckpt from {}/best_val.pth.tar".format(artifact_dir))
        self.model = PointNetCls(sd, device=device)
        assert self.model.n_out == n_out, f"checkpoint has {self.model.n_out} classes, config says {n_out}"
        self.subsample = "host"       # "host": the reference's numpy draw, bit for bit; "device": counter-based draw on the GPU
        self.chunk = 1024             # candidates per pipeline stage (host draw of chunk k+1 overlaps the GPU on chunk k)
        self._pin = None
        self.engine = self._pick_engine() if engine == "auto" else int(engine)

    def _pick_engine(self):
        """Engine 3 rounds the 128->1024 layer's operands to fp16.  With THIS checkpoint's weights, score a seeded probe
        batch (64 unit-scale clouds of n_pts points, private RandomState: the global numpy generator is untouched) on
        engine 3 and on the near-fp32 engine 1; keep engine 3 only if every probability agrees within ENGINE_TOL and no
        activation left the fp16 range -- otherwise this predicter runs on engine 1 (about 1.8x slower)."""
        net = self.model
        ctx = net.ctx
        keep = ctx.get_engine()
        n = min(int(self.cfg["n_pts"]), 1024)
        x = np.random.RandomState(20240923).normal(0.0, 1.0, (64, n, 6)).astype(np.float32)
        out = {}
        try:
            for e in (1, 3):
                ctx.set_engine(e)
                ctx.fp16_overflow()
                out[e] = net.forward(x, return_probs=True)[1].cpu().numpy()
            clamped = ctx.fp16_overflow()
        finally:
            ctx.set_engine(keep)
        dev = float(np.abs(out[1] - out[3]).max())
        self.engine_probe = {"max_abs_dprob": dev, "fp16_clamp": bool(clamped)}
        return 3 if (dev <= self.ENGINE_TOL and not clamped) else 1

    def _pinned_ids(self, B, n_pts):
        import torch
        need = B * n_pts
        if self._pin is None or self._pin.numel() < need:
            self._pin = torch.empty((need + need // 4,), dtype=torch.int32).pin_memory()
        return self._pin[:need].view(B, n_pts)

    def predict_batch(self, data, grasp_poses, ids=None, subsample=None, shard=None):
        """predicter.py:67-94.  Returns list of [label np.int64, confidence np.float32, probs (n_out,) f32].

        ``data`` is not modified (the reference deep-copies it, :72).  ``ids`` (B,n_pts) overrides the draw.
        ``subsample`` (default ``self.subsample``):
          "host"   -- the reference's per-candidate ``np.random.choice`` (dataset_grasp.py:72-73), bit for bit and
                      with the same consumption of the global numpy generator; drawn in C in chunks on a worker thread
                      while the GPU scores the previous chunk;
          "device" -- a statistically equivalent counter-based draw on the GPU (cg_draw_ids_dev); consumes ONE value
                      of the global numpy generator (the seed) instead of one shuffle per candidate.  Not the
                      reference's numbers: use it when throughput matters more than replaying a reference run.
        ``shard=(lo, hi)`` scores only candidates [lo, hi) of the list and returns their (hi-lo, n_out) probabilities
        as a CUDA tensor -- the random stream is consumed for the WHOLE list (the other candidates' draws are skipped in
        C), so every rank of a sharded call stays on the reference's stream (catgrasp_b200.dist.sharded_predict_batch).
        """
        import torch
        from . import _lib
        B_all = len(grasp_poses)
        if B_all == 0:
            return []
        lo_s, hi_s = (0, B_all) if shard is None else (int(shard[0]), int(shard[1]))
        assert 0 <= lo_s <= hi_s <= B_all
        B = hi_s - lo_s
        mode = subsample or self.subsample
        assert mode in ("host", "device"), mode
        xyz = np.asarray(data["cloud_xyz"], dtype=np.float64)
        nrm = np.asarray(data["cloud_normal"], dtype=np.float64)
        valid_mask = xyz[:, 2] >= 0.1                                   # dataset_grasp.py:64
        xyz = np.ascontiguousarray(xyz[valid_mask].reshape(-1, 3))
        nrm = np.ascontiguousarray(nrm[valid_mask].reshape(-1, 3))
        M, n_pts = xyz.shape[0], int(self.cfg["n_pts"])
        poses = np.ascontiguousarray(np.asarray(grasp_poses, dtype=np.float64).reshape(B_all, 4, 4)[lo_s:hi_s])
        if ids is not None:
            ids = np.asarray(ids)[lo_s:hi_s]
        net, dev = self.model, self.model.device
        ctx_engine = net.ctx.get_engine()
        if ctx_engine != self.engine:       # the context (one per device) is shared: select this predicter's engine per call
            net.ctx.set_engine(self.engine)
        try:
            return self._predict_batch(data, grasp_poses, ids, mode, shard, xyz, nrm, poses, M, n_pts, B, B_all, lo_s, hi_s)
        finally:
            if ctx_engine != self.engine:
                net.ctx.set_engine(ctx_engine)

    def _predict_batch(self, data, grasp_poses, ids, mode, shard, xyz, nrm, poses, M, n_pts, B, B_all, lo_s, hi_s):
        import torch
        net, dev = self.model, self.model.device
        if B == 0:   # an empty shard still consumes the stream like everybody else
            if ids is None and mode == "device":
                np.random.randint(0, 2 ** 63 - 1, dtype=np.int64)
            elif ids is None:
                d = _LegacyDraw()
                d.skip(M, n_pts, B_all)
                d.commit()
            import torch as _t
            return _t.empty((0, net.n_out), dtype=_t.float32, device=dev)
        with torch.cuda.device(dev):
            d_xyz, d_nrm = torch.from_numpy(xyz).to(dev), torch.from_numpy(nrm).to(dev)
            d_pose = torch.from_numpy(poses).to(dev)
            d_mean = torch.from_numpy(np.ascontiguousarray(self.cfg["mean"].reshape(-1))).to(dev) if "mean" in self.cfg else None
            d_std = torch.from_numpy(np.ascontiguousarray(self.cfg["std"].reshape(-1))).to(dev) if "std" in self.cfg else None
            d_probs = torch.empty((B, net.n_out), dtype=torch.float32, device=dev)
            d_label = torch.empty((B,), dtype=torch.int32, device=dev)

            def run(engine_override=None):
                if ids is not None or mode == "device":
                    if ids is not None:
                        d_ids = torch.from_numpy(np.ascontiguousarray(ids, dtype=np.int32)).to(dev)
                    else:
                        d_ids = net.draw_ids_dev(M, n_pts, B, seed=self._device_seed, first_candidate=lo_s)
                    net.graspq_dev(d_xyz, d_nrm, d_pose, d_ids, d_mean, d_std, out=(d_probs, d_label))
                    return
                # bit-parity mode: C continuation of numpy's generator on a worker thread, chunk by chunk
                import queue
                import threading
                h_ids = self._pinned_ids(B, n_pts)
                draw = self._draw
                bounds = [(lo, min(B, lo + self.chunk)) for lo in range(0, B, self.chunk)]
                q = queue.Queue()

                def producer():
                    try:
                        if not self._drawn and lo_s > 0:
                            draw.skip(M, n_pts, lo_s)
                        for lo, hi in bounds:
                            if not self._drawn:
                                draw.draw(M, n_pts, hi - lo, out=h_ids[lo:hi])
                            q.put((lo, hi))
                        if not self._drawn and hi_s < B_all:
                            draw.skip(M, n_pts, B_all - hi_s)
                    except Exception as e:   # surfaces in the consumer
                        q.put(e)
                t = threading.Thread(target=producer, daemon=True)
                t.start()
                d_ids = torch.empty((B, n_pts), dtype=torch.int32, device=dev)
                for _ in bounds:
                    item = q.get()
                    if isinstance(item, Exception):
                        raise item
                    lo, hi = item
                    d_ids[lo:hi].copy_(h_ids[lo:hi], non_blocking=True)
                    net.graspq_dev(d_xyz, d_nrm, d_pose[lo:hi], d_ids[lo:hi], d_mean, d_std,
                                   out=(d_probs[lo:hi], d_label[lo:hi]))
                t.join()
                self._drawn = True

            if ids is None and mode == "device":
                self._device_seed = int(np.random.randint(0, 2 ** 63 - 1, dtype=np.int64))
            if ids is None and mode == "host":
                self._draw, self._drawn = _LegacyDraw(), False
            run()
            probs = None if shard is not None else d_probs.cpu().numpy()
            if net.ctx.get_engine() >= 2 and net.ctx.fp16_overflow():
                # the fast engines clamp the 128->1024 layer's inputs to the fp16 range: redo on the near-fp32 engine
                print("GraspPredicter: activation beyond the fp16 range, re-running on engine 1 (wgmma bf16 hi/lo x3)")
                eng = net.ctx.get_engine()
                net.ctx.set_engine(1)
                try:
                    run()
                    probs = None if shard is not None else d_probs.cpu().numpy()
                finally:
                    net.ctx.set_engine(eng)
            if ids is None and mode == "host":
                self._draw.commit()
        if shard is not None:
            return d_probs
        labels = probs.argmax(1)                                         # predicter.py:87-91
        conf = probs[np.arange(B), labels]
        return [[l, c, p] for l, c, p in zip(labels, conf, probs)]


class NunocsPredicter:
    """predicter.py:98-203."""

    class_name_to_artifact_id = {"nut": 78, "hnm": 73, "screw": 76}

    def __init__(self, class_name, artifact_dir=None, device=None):
        self.class_name = class_name
        if class_name == "nut":                                         # predicter.py:106-114
            self.min_scale = [0.005, 0.005, 0.001]
            self.max_scale = [0.05, 0.05, 0.05]
        else:
            self.min_scale = [0.005, 0.005, 0.005]
            self.max_scale = [0.15, 0.05, 0.05]
        artifact_id = self.class_name_to_artifact_id[class_name]
        if artifact_dir is None:
            artifact_dir = f"{_CODE_DIR}/artifacts/artifacts-{artifact_id}"
        print("NunocsPredicter artifact_dir", artifact_dir)
        self.cfg = _load_artifacts(artifact_dir, "config_nunocs.yml")
        sd = load_checkpoint(f"{artifact_dir}/best_val.pth.tar")
        self.model = PointNetSeg(sd, device=device)
        assert self.model.n_out == 3 * self.cfg["ce_loss_bins"]
        self.ransac_max_iter = 10000

    def transform(self, data, ids=None):
        """NunocsIsolatedDataset.transform in 'test' phase (dataset_nunocs.py:38-65)."""
        keep_ids = np.arange(data["cloud_xyz"].shape[0])
        valid_mask = data["cloud_xyz"][:, 2] >= 0.1
        keep_ids = keep_ids[valid_mask]
        data["cloud_xyz"] = data["cloud_xyz"][valid_mask]
        if ids is None:
            ids = draw_subsample_ids(data["cloud_xyz"].shape[0], int(self.cfg["n_pts"]))
        data["cloud_xyz"] = data["cloud_xyz"][ids]
        keep_ids = keep_ids[ids]
        data["cloud_nocs"] = data["cloud_nocs"][keep_ids].reshape(-1, 3) / 255.0
        data["cloud_rgb"] = data["cloud_rgb"][keep_ids].reshape(-1, 3)
        data["cloud_normal"] = data["cloud_normal"][keep_ids].reshape(-1, 3)
        data["cloud_xyz_original"] = copy.deepcopy(data["cloud_xyz"])
        data["keep_ids"] = keep_ids
        max_xyz = data["cloud_xyz"].max(axis=0)                         # augmentations.py:70-75
        min_xyz = data["cloud_xyz"].min(axis=0)
        scale = (max_xyz - min_xyz).max()
        data["cloud_xyz"] = (data["cloud_xyz"] - min_xyz) / (scale + 1e-15)
        data["input"] = np.concatenate((data["cloud_xyz"], data["cloud_normal"]), axis=-1)
        if "mean" in self.cfg:
            data["input"] = (data["input"] - self.cfg["mean"].reshape(1, -1)) / (self.cfg["std"].reshape(1, -1) + 1e-15)
        if "color_file" in data:
            del data["color_file"]
        return data

    def predict_nocs(self, data, ids=None):
        """Network half of predict (predicter.py:136-150): returns (nocs_cloud (N,3) f32, confidence_z (N,))."""
        data["cloud_nocs"] = np.zeros(data["cloud_xyz"].shape)
        data["cloud_rgb"] = np.zeros(data["cloud_xyz"].shape)
        data_transformed = self.transform(copy.deepcopy(data), ids=ids)
        self.data_transformed = data_transformed
        x = np.ascontiguousarray(data_transformed["input"], dtype=np.float64).astype(np.float32)
        coords, conf_z, bins = self.model.nunocs_host(x, int(self.cfg["ce_loss_bins"]))
        self.confidence_z = conf_z
        self.pred_bins = bins
        return coords, conf_z

    def predict(self, data, ids=None):
        """predicter.py:135-203: (nocs_cloud, transform) or (None, None)."""
        from .aligning import estimate9DTransform
        nocs_cloud, _ = self.predict_nocs(data, ids=ids)
        ori_cloud = self.data_transformed["cloud_xyz_original"]
        nocs_cloud_down = copy.deepcopy(nocs_cloud)
        ori_cloud_down = copy.deepcopy(ori_cloud)
        best_ratio = 0
        best_transform = None
        best_symmetry_tf = None
        for symmetry_tf in [np.eye(4)]:
            tmp_nocs_cloud_down = (symmetry_tf @ to_homo(nocs_cloud_down).T).T[:, :3]
            for thres in [0.003, 0.005]:
                transform, inliers = estimate9DTransform(
                    source=tmp_nocs_cloud_down, target=ori_cloud_down, PassThreshold=thres,
                    max_iter=self.ransac_max_iter, max_scale=self.max_scale, min_scale=self.min_scale,
                    max_dimensions=np.array([1.2, 1.2, 1.2]))
                if transform is None:
                    continue
                if np.linalg.det(transform[:3, :3]) < 0:
                    continue
                transformed = (transform @ to_homo(tmp_nocs_cloud_down).T).T[:, :3]
                err_thres = 0.003
                errs = np.linalg.norm(transformed - ori_cloud_down, axis=1)
                ratio = np.sum(errs <= err_thres) / len(errs)
                if ratio > best_ratio:
                    best_ratio = ratio
                    best_symmetry_tf = symmetry_tf
                    best_transform = transform.copy()
        if best_transform is None:
            return None, None
        self.best_ratio = best_ratio
        transform = best_transform
        self.nocs_pose = transform.copy()
        nocs_cloud = (best_symmetry_tf @ to_homo(nocs_cloud).T).T[:, :3]
        return nocs_cloud, transform


def flatten_config(cfg, out=None):
    """PointGroup/util/config.py key_to_attr: every leaf of the nested config sections as one flat dict (a later
    section's key overwrites an earlier one's, as setattr does)."""
    out = {} if out is None else out
    for k, v in cfg.items():
        if isinstance(v, dict):
            flatten_config(v, out)
        else:
            out[k] = v
    return out


def slice_keep_mask(xyz):
    """predicter.py:246-249 with n_slice_per_side = 1, in the input's dtype as the reference writes it: in float32
    xmin + (xmax - xmin) can round below xmax, and a point at xmax is then dropped."""
    x, y = xyz[:, 0], xyz[:, 1]
    xmin, xmax, ymin, ymax = x.min(), x.max(), y.min(), y.max()
    xlen, ylen = (xmax - xmin) / 1, (ymax - ymin) / 1
    return (x >= xmin) & (x <= xmin + xlen) & (y >= ymin) & (y <= ymin + ylen)


class PointGroupPredictor:
    """predicter.py:206-338: the segmentation of a pile into instances.  The front runs on the device's cloud kernels
    (device_front), the network (voxelisation, U-Net, offset head) on the device (catgrasp_b200.pointgroup),
    the clustering after it in segment.pointgroup_labels.  Only the shipped structure is implemented: mode 4,
    use_coords, residual blocks, input_channel 3 and n_slice_per_side 1; any m and block_reps 1 or 2."""

    class_name_to_artifact_id = {"nut": 40, "hnm": 68, "screw": 77}

    def __init__(self, class_name, artifact_dir=None, device=None):
        from .pointgroup import PointGroupNet
        from .segment import MEANSHIFT_BANDWIDTH
        if class_name not in MEANSHIFT_BANDWIDTH:
            raise NotImplementedError(f"PointGroupPredictor: no clustering bandwidth for class {class_name!r}")
        self.class_name = class_name
        if artifact_dir is None:
            artifact_dir = f"{_CODE_DIR}/artifacts/artifacts-{self.class_name_to_artifact_id[class_name]}"
        print("PointGroupPredictor artifact_dir", artifact_dir)
        with open(f"{artifact_dir}/config_pointgroup.yaml", "r") as ff:
            self.cfg = yaml.safe_load(ff)
        self.cfg_pg = flatten_config(self.cfg)
        self.n_slice_per_side = 1
        self._check_structure()
        sd = load_checkpoint(f"{artifact_dir}/best_val.pth.tar")
        self.model = PointGroupNet(sd, int(self.cfg_pg["m"]), int(self.cfg_pg["block_reps"]), device=device)

    def _check_structure(self):
        c = self.cfg_pg
        for key, want in (("mode", 4), ("use_coords", True), ("block_residual", True), ("input_channel", 3)):
            if c.get(key) != want:
                raise NotImplementedError(f"PointGroupPredictor: {key} = {c.get(key)!r}; only the shipped {key} = "
                                          f"{want!r} is implemented")
        if self.n_slice_per_side != 1:
            raise NotImplementedError("PointGroupPredictor: n_slice_per_side must be 1 (the site tables hold one "
                                      "batch)")
        if int(c["block_reps"]) not in (1, 2):
            raise NotImplementedError(f"PointGroupPredictor: block_reps = {c['block_reps']}; only 1 and 2 build")

    def device_front(self, data):
        """predicter.py:234-300 with n_slice_per_side = 1, on the device for numpy or CUDA input: (xyz_original_all
        (N,3) float32, locs (N,3) int64, feats (N,6) float32) CUDA tensors and spatial_shape (3 ints).  Every step is
        in the input's dtype as the reference computes it: the keep mask, the 0.5 mm voxel means snapped to their
        nearest point, and the sites trunc(fl(fl(x * scale) - min)), the scale first and each operation rounded on
        its own."""
        import torch
        from .cloud import CloudIndex
        from . import _lib
        self._check_structure()
        dev = self.model.ctx.device
        ctx, xyz, nrm = _lib.inputs(data["cloud_xyz"], data["cloud_normal"], ctx=self.model.ctx,
                                    dtype=tuple(_float_dtype(a) for a in (data["cloud_xyz"], data["cloud_normal"])))
        keep = torch.nonzero(slice_keep_mask(xyz)).reshape(-1)
        xo, no = xyz[keep], nrm[keep]
        ds = float(self.cfg["downsample_size"])
        down, _ = CloudIndex(xo, ds, dev).voxel_means()
        # the snap (cKDTree.query): a voxel mean and its members share a voxel, so the nearest member is within the
        # diagonal, widened by 1e-9 relative against rounding at a voxel face
        snap = ds * np.sqrt(3.0) * (1 + 1e-9)
        _, ids = CloudIndex(xo, snap, dev).nearest(down, snap)
        if bool((ids < 0).any()):
            raise _lib.CgError("PointGroupPredictor: a voxel mean has no point within its voxel's diagonal")
        ids = ids.to(torch.int64)
        xo, no = xo[ids], no[ids]
        s = xo * self.cfg_pg["scale"]
        s = s - s.amin(0)
        locs = s.to(torch.int64)                                         # truncation, as torch's .long() on the host
        hi = (locs.amax(0) + 1).cpu().numpy()
        shape = tuple(int(v) for v in np.maximum(hi, int(self.cfg_pg["full_scale"][0])))
        feats = torch.cat([no.to(torch.float32), xo.to(torch.float32)], 1)
        return xo.to(torch.float32), locs, feats, shape

    def host_front(self, data):
        """device_front with numpy results: (xyz_original_all (N,3) float32, locs (N,3) int64, feats (N,6) float32,
        spatial_shape (3 ints))."""
        xo, locs, feats, shape = self.device_front(data)
        return xo.cpu().numpy(), locs.cpu().numpy(), feats.cpu().numpy(), shape

    def offsets(self, data):
        """The front and the network: (xyz_original_all (N,3) float32, pt_offsets (N,3) float32), CUDA tensors."""
        from . import spconv
        xo, locs, feats, shape = self.device_front(data)
        level, p2v = spconv.index(locs, shape)
        return xo, self.model.offsets(level, p2v, feats)

    def predict(self, data):
        """predicter.py:232-338: labels_all (M,) int64, one per point of data['cloud_xyz'], and self.xyz_shifted; numpy
        for numpy input, CUDA tensors for CUDA input."""
        from .segment import MEANSHIFT_BANDWIDTH, pointgroup_labels
        xo, off = self.offsets(data)
        labels_all, xyz_shifted = pointgroup_labels(xo, off, data["cloud_xyz"], MEANSHIFT_BANDWIDTH[self.class_name])
        if not getattr(data["cloud_xyz"], "is_cuda", False):
            labels_all, xyz_shifted = labels_all.cpu().numpy(), xyz_shifted.cpu().numpy()
        self.xyz_shifted = xyz_shifted
        return labels_all


def _float_dtype(a):
    """torch dtype of a float32 / float64 array or tensor (anything else is widened to float64)."""
    import torch
    name = str(a.dtype)
    return torch.float32 if name.endswith("float32") else torch.float64
