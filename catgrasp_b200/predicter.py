"""GraspPredicter / NunocsPredicter with the reference's call surface (predicter.py:39-203).

Host side (numpy, identical RNG consumption to the reference):
  * z >= 0.1 mask and the per-candidate ``np.random.choice`` subset (dataset_grasp.py:64,72-73;
    dataset_nunocs.py:40-44) -- only the *indices* are drawn on the host;
  * NUNOCS min/max-extent normalisation (augmentations.py:70-75);
  * the 9-DoF RANSAC's 4-subsets (aligning.py:91-97), drawn in C on numpy's generator.
Device side (libcatgrasp_b200.so): per-candidate rigid transform + normalisation + PointNet forward
+ softmax / argmax post-processing; the 9-DoF RANSAC's scoring and selection at both thresholds (one launch).
``subsample = "device"`` on either predicter moves the draws (and NUNOCS's transform) to the GPU as well.
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


def draw_nunocs_many(Ms, n_pts, n_hyp, given=None):
    """The host-mode random numbers of a loop of NunocsPredicter.predict calls, in the loop's order, in one walk of
    numpy's GLOBAL generator (cg_host_legacy_choice): for each object b, its cloud subset
    ``np.random.choice(np.arange(Ms[b]), n_pts, replace=Ms[b] < n_pts)`` (not drawn where ``given[b]`` is not None),
    then its ``n_hyp`` RANSAC 4-subsets of n_pts points (aligning.py:91-97).  Returns (list of (n_pts,) int32 subsets
    or None, (B, n_hyp, 4) int32); the generator's state is put back once, at the end."""
    B = len(Ms)
    hyp = np.empty((B, n_hyp, 4), dtype=np.int32)
    subs = []
    d = _LegacyDraw()
    for b, M in enumerate(Ms):
        subs.append(d.draw(int(M), n_pts, 1)[0] if given is None or given[b] is None else None)
        d.draw(n_pts, 4, n_hyp, out=hyp[b])
    d.commit()
    return subs, hyp


GRASPQ_CHUNK_B = 16384   # candidates per internal pass of cg_graspq_forward_*_dev (CG_GRASPQ_CHUNK_B)


def graspq_fc_groups(counts, launch=None):
    """The FC row groups of a loop of GraspPredicter.score calls, one per object with counts[o] candidates: each
    call's graspq_dev launches cover ``launch`` candidates (host-drawn subsets: GraspPredicter.chunk) or the whole
    list (None: device-drawn or given subsets), and cg_graspq_forward_dev cuts each launch at GRASPQ_CHUNK_B.
    Returns (groups (G,) int32 row counts in row order, spans (O,2) int64: object o's groups are
    groups[spans[o,0]:spans[o,1]])."""
    groups, spans = [], np.zeros((len(counts), 2), np.int64)
    for o, B in enumerate(counts):
        spans[o, 0] = len(groups)
        step = B if launch is None else int(launch)
        for c0 in range(0, B, max(step, 1)):
            L = min(step, B - c0)
            groups += [min(GRASPQ_CHUNK_B, L - k) for k in range(0, L, GRASPQ_CHUNK_B)]
        spans[o, 1] = len(groups)
    return np.asarray(groups, np.int32), spans


def host_draw_stages(groups, chunk):
    """Stages of the host-drawn pipeline: consecutive groups packed into row ranges of at most ``chunk`` rows (one
    group per stage where a group is larger).  Returns a list of (first row, end row, first group, end group)."""
    stages, r0, g0, rows = [], 0, 0, 0
    for g, m in enumerate(groups):
        if rows and rows + int(m) > chunk:
            stages.append((r0, r0 + rows, g0, g))
            r0, g0, rows = r0 + rows, g, 0
        rows += int(m)
    if rows:
        stages.append((r0, r0 + rows, g0, len(groups)))
    return stages


def walk_grasp_many(Ms, counts, n_pts, stages, out):
    """The host-mode draws of a loop of GraspPredicter.predict_batch calls in ONE walk of numpy's global generator
    (cg_host_legacy_choice): object o's counts[o] subsets of n_pts points out of Ms[o] (replace = Ms[o] < n_pts), in
    object order, into the rows of ``out`` (sum(counts), n_pts) int32.  A generator: it draws stage by stage (row
    ranges from host_draw_stages, cut anywhere) and yields each stage as it is drawn; the generator's state is put
    back once, after the last stage."""
    draw = _LegacyDraw()
    first = np.concatenate([[0], np.cumsum(np.asarray(counts, np.int64))])
    for stage in stages:
        r0, r1 = int(stage[0]), int(stage[1])
        o = int(np.searchsorted(first, r0, side="right")) - 1
        r = r0
        while r < r1:
            while first[o + 1] <= r:
                o += 1
            e = min(r1, int(first[o + 1]))
            draw.draw(int(Ms[o]), n_pts, e - r, out=out[r:e])
            r = e
        yield stage
    draw.commit()


def _check_grasp_many(datas, grasp_poses_list, ids, n_pts):
    """predict_batch_many's checks, before any draw: per object (masked xyz (M,3) f64, masked normals, poses (B,4,4)
    f64, ids (B,n_pts) int32 or None), or None for an object with no candidates (predict_batch returns [] for it
    without looking at its data).  ValueError for anything predict_batch would fail on, and for ids outside the
    object's masked cloud."""
    datas, grasp_poses_list = list(datas), list(grasp_poses_list)
    if len(grasp_poses_list) != len(datas):
        raise ValueError(f"predict_batch_many: {len(grasp_poses_list)} pose lists for {len(datas)} objects")
    if ids is not None and len(ids) != len(datas):
        raise ValueError(f"predict_batch_many: {len(ids)} id arrays for {len(datas)} objects")
    out = []
    for o, (data, grasps) in enumerate(zip(datas, grasp_poses_list)):
        B = len(grasps)
        if B == 0:
            out.append(None)
            continue
        poses = np.asarray(grasps, dtype=np.float64)
        if poses.size != B * 16:
            raise ValueError(f"predict_batch_many: object {o} has {B} poses of {poses.size // B} values, not 4x4")
        if not hasattr(data, "keys") or "cloud_xyz" not in data or "cloud_normal" not in data:
            raise ValueError(f"predict_batch_many: object {o} is not a dict with 'cloud_xyz' and 'cloud_normal'")
        xyz = np.asarray(data["cloud_xyz"], dtype=np.float64)
        nrm = np.asarray(data["cloud_normal"], dtype=np.float64)
        if xyz.ndim != 2 or xyz.shape[1] != 3 or nrm.shape != xyz.shape:
            raise ValueError(f"predict_batch_many: object {o} has cloud_xyz {xyz.shape} and cloud_normal {nrm.shape}; "
                             f"both must be (M,3)")
        valid_mask = xyz[:, 2] >= 0.1                                   # dataset_grasp.py:64
        xyz, nrm = np.ascontiguousarray(xyz[valid_mask]), np.ascontiguousarray(nrm[valid_mask])
        if xyz.shape[0] == 0:
            raise ValueError("'a' cannot be empty unless no samples are taken")   # predict_batch's np.random.choice
        sub = None
        if ids is not None:
            sub = np.asarray(ids[o])
            if sub.shape != (B, n_pts):
                raise ValueError(f"predict_batch_many: ids[{o}] has shape {sub.shape}, not ({B}, {n_pts})")
            if sub.min() < 0 or sub.max() >= xyz.shape[0]:
                raise ValueError(f"predict_batch_many: ids[{o}] indexes outside the {xyz.shape[0]} points with "
                                 f"z >= 0.1")
            sub = sub.astype(np.int32)
        out.append((xyz, nrm, poses.reshape(B, 4, 4), sub))
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

    def _given_ids(self, ids, lo, hi):
        """Caller-given subsets: numpy's global generator is not touched.  Yields (first row, device ids) launches."""
        import torch
        if hi > lo:
            yield 0, torch.from_numpy(np.ascontiguousarray(np.asarray(ids)[lo:hi], dtype=np.int32)).to(self.model.device)

    def _device_draw(self, M, lo, hi):
        """The counter-based draw on the GPU (cg_draw_ids_dev): consumes ONE value of numpy's global generator, the
        seed, whatever the shard; a candidate's subset depends on the seed and its place in the whole list only."""
        seed = int(np.random.randint(0, 2 ** 63 - 1, dtype=np.int64))
        if hi > lo:
            yield 0, self.model.draw_ids_dev(M, int(self.cfg["n_pts"]), hi - lo, seed=seed, first_candidate=lo)

    def _host_draw(self, M, lo, hi, B_all):
        """The reference's draw: walks numpy's global generator over the WHOLE list in C (skip the ``lo`` candidates
        before the shard, draw the shard, skip the ``B_all - hi`` after it) and puts the advanced state back.  The
        worker thread draws chunk k+1 into the pinned buffer while the GPU scores chunk k."""
        import queue
        import threading
        import torch
        B, n_pts = hi - lo, int(self.cfg["n_pts"])
        h_ids = self._pinned_ids(B, n_pts)
        d_ids = torch.empty((B, n_pts), dtype=torch.int32, device=self.model.device)
        draw = _LegacyDraw()
        q = queue.Queue()

        def producer():
            try:
                draw.skip(M, n_pts, lo)
                for c0 in range(0, B, self.chunk):
                    c1 = min(B, c0 + self.chunk)
                    draw.draw(M, n_pts, c1 - c0, out=h_ids[c0:c1])
                    q.put((c0, c1))
                draw.skip(M, n_pts, B_all - hi)
                q.put(None)
            except Exception as e:   # surfaces in the consumer
                q.put(e)
        t = threading.Thread(target=producer, daemon=True)
        t.start()
        while (item := q.get()) is not None:
            if isinstance(item, Exception):
                raise item
            c0, c1 = item
            d_ids[c0:c1].copy_(h_ids[c0:c1], non_blocking=True)
            yield c0, d_ids[c0:c1]
        t.join()
        draw.commit()

    def score(self, data, grasp_poses, ids=None, subsample=None, shard=None):
        """The probabilities of candidates ``shard=(lo, hi)`` of the list (default: all of it) as a (hi-lo, n_out)
        float32 CUDA tensor.

        ``data`` is not modified (the reference deep-copies it, :72).  ``ids`` (B,n_pts) overrides the draw.
        ``subsample`` (default ``self.subsample``):
          "host"   -- the reference's per-candidate ``np.random.choice`` (dataset_grasp.py:72-73), bit for bit and
                      with the same consumption of the global numpy generator; drawn in C in chunks on a worker thread
                      while the GPU scores the previous chunk;
          "device" -- a statistically equivalent counter-based draw on the GPU (cg_draw_ids_dev); consumes ONE value
                      of the global numpy generator (the seed) instead of one shuffle per candidate.  Not the
                      reference's numbers: use it when throughput matters more than replaying a reference run.
        The random stream is consumed for the WHOLE list whatever the shard, so every rank of a sharded call stays on
        the reference's stream (catgrasp_b200.dist.sharded_predict_batch).
        """
        import torch
        B_all = len(grasp_poses)
        lo, hi = (0, B_all) if shard is None else (int(shard[0]), int(shard[1]))
        assert 0 <= lo <= hi <= B_all
        mode = subsample or self.subsample
        assert mode in ("host", "device"), mode
        xyz = np.asarray(data["cloud_xyz"], dtype=np.float64)
        nrm = np.asarray(data["cloud_normal"], dtype=np.float64)
        valid_mask = xyz[:, 2] >= 0.1                                   # dataset_grasp.py:64
        xyz = np.ascontiguousarray(xyz[valid_mask].reshape(-1, 3))
        nrm = np.ascontiguousarray(nrm[valid_mask].reshape(-1, 3))
        M = xyz.shape[0]
        poses = np.ascontiguousarray(np.asarray(grasp_poses, dtype=np.float64).reshape(B_all, 4, 4)[lo:hi])
        net, dev, ctx = self.model, self.model.device, self.model.ctx
        with torch.cuda.device(dev):
            d_xyz, d_nrm = torch.from_numpy(xyz).to(dev), torch.from_numpy(nrm).to(dev)
            d_pose = torch.from_numpy(poses).to(dev)
            d_mean = torch.from_numpy(np.ascontiguousarray(self.cfg["mean"].reshape(-1))).to(dev) if "mean" in self.cfg else None
            d_std = torch.from_numpy(np.ascontiguousarray(self.cfg["std"].reshape(-1))).to(dev) if "std" in self.cfg else None
            d_probs = torch.empty((hi - lo, net.n_out), dtype=torch.float32, device=dev)
            d_label = torch.empty((hi - lo,), dtype=torch.int32, device=dev)

            def forward(c0, d_ids):
                c1 = c0 + d_ids.shape[0]
                net.graspq_dev(d_xyz, d_nrm, d_pose[c0:c1], d_ids, d_mean, d_std, out=(d_probs[c0:c1], d_label[c0:c1]))

            if ids is not None:
                launches = self._given_ids(ids, lo, hi)
            elif mode == "device":
                launches = self._device_draw(M, lo, hi)
            else:
                launches = self._host_draw(M, lo, hi, B_all)
            ctx_engine = ctx.get_engine()
            ctx.set_engine(self.engine)         # the context (one per device) is shared: this predicter's engine, per call
            try:
                done = []
                for c0, d_ids in launches:
                    forward(c0, d_ids)
                    done.append((c0, d_ids))
                if self.engine >= 2 and ctx.fp16_overflow():
                    # the fast engines clamp the 128->1024 layer's inputs to the fp16 range: redo on the near-fp32
                    # engine from the ids already on the device, launch for launch (a launch's batch size selects the
                    # FC kernel, so the same cuts give the bits of a call made on engine 1)
                    print("GraspPredicter: activation beyond the fp16 range, re-running on engine 1 (wgmma bf16 hi/lo x3)")
                    ctx.set_engine(1)
                    for c0, d_ids in done:
                        forward(c0, d_ids)
            finally:
                ctx.set_engine(ctx_engine)
        return d_probs

    def predict_batch(self, data, grasp_poses, ids=None, subsample=None):
        """predicter.py:67-94.  Returns list of [label np.int64, confidence np.float32, probs (n_out,) f32]: ``score``
        on the whole list (same ``ids`` and ``subsample``), copied to the host once."""
        if len(grasp_poses) == 0:
            return []
        return result_list(self.score(data, grasp_poses, ids=ids, subsample=subsample).cpu().numpy())

    def score_many(self, datas, grasp_poses_list, ids=None, subsample=None):
        """``score`` for several objects, each with its own cloud and candidate list, in one pass: (probs (sum B_o,
        n_out) float32 CUDA tensor, offsets (O+1,) int64), object o's rows probs[offsets[o]:offsets[o+1]] equal bit for
        bit to ``score(datas[o], grasp_poses_list[o], ids[o], subsample)`` in a loop over the objects that skips those
        with no candidates (as predict_batch does), from the same numpy state, which it leaves where the loop would.

        ``datas`` are numpy dicts, not modified; ``ids`` (optional) a list of per-object (B_o, n_pts) subsets.  The
        random numbers are the loop's:
          "host"   -- one walk of numpy's global generator over all objects' subsets, in object order, drawn on a
                      worker thread stage by stage (about ``chunk`` candidates) while the GPU scores the previous stage;
          "device" -- one np.random.randint seed per object with candidates, and one cg_draw_ids_many_dev launch.
        The FC layers run on the loop's launches (graspq_fc_groups): host mode ``chunk`` candidates per launch, device
        and given-ids modes the object's whole list, cut at GRASPQ_CHUNK_B.  The whole list is checked before anything
        is drawn: on a ValueError numpy's generator is untouched.

        On engines 2 and 3 the fp16-overflow flag belongs to the context: when it is set after the pass (or was set
        before it, which the loop's first call would see), the objects are scored again one at a time from the ids on
        the device, each on this predicter's engine and, where that object overflows, on engine 1, as the loop does."""
        import torch
        mode = subsample or self.subsample
        assert mode in ("host", "device"), mode
        n_pts = int(self.cfg["n_pts"])
        objs = _check_grasp_many(datas, grasp_poses_list, ids, n_pts)
        counts = [0 if ob is None else ob[2].shape[0] for ob in objs]
        offsets = np.zeros(len(objs) + 1, np.int64)
        offsets[1:] = np.cumsum(counts)
        B_all = int(offsets[-1])
        live = [o for o, ob in enumerate(objs) if ob is not None]
        Ms = [0 if ob is None else ob[0].shape[0] for ob in objs]
        bases = np.zeros(len(objs), np.int64)
        bases[1:] = np.cumsum(Ms)[:-1]
        if sum(Ms) >= 2 ** 31:
            raise ValueError("predict_batch_many: 2^31 cloud points or more in all")
        launch = self.chunk if (ids is None and mode == "host") else None
        groups, spans = graspq_fc_groups(counts, launch)
        net, dev, ctx = self.model, self.model.device, self.model.ctx
        with torch.cuda.device(dev):
            d_probs = torch.empty((B_all, net.n_out), dtype=torch.float32, device=dev)
            if B_all == 0:
                return d_probs, offsets
            cat = lambda k: np.ascontiguousarray(np.concatenate([objs[o][k] for o in live]))
            d_xyz, d_nrm, d_pose = (torch.from_numpy(cat(k)).to(dev) for k in (0, 1, 2))
            d_mean = torch.from_numpy(np.ascontiguousarray(self.cfg["mean"].reshape(-1))).to(dev) if "mean" in self.cfg else None
            d_std = torch.from_numpy(np.ascontiguousarray(self.cfg["std"].reshape(-1))).to(dev) if "std" in self.cfg else None

            def forward(r0, r1, g0, g1, d_ids):
                net.graspq_many_dev(d_xyz, d_nrm, d_pose[r0:r1], d_ids[r0:r1], groups[g0:g1], d_mean, d_std,
                                    out=(d_probs[r0:r1], None))

            whole = [(0, B_all, 0, len(groups))]
            if ids is not None:
                d_ids = torch.from_numpy(np.concatenate([objs[o][3] + np.int32(bases[o]) for o in live])).to(dev)
                stages = iter(whole)
            elif mode == "device":
                seeds = [int(np.random.randint(0, 2 ** 63 - 1, dtype=np.int64)) for _ in live]
                d_ids = net.draw_ids_many_dev([Ms[o] for o in live], n_pts, [counts[o] for o in live], seeds,
                                              bases[live])
                stages = iter(whole)
            else:
                h_ids = self._pinned_ids(B_all, n_pts)
                d_ids = torch.empty((B_all, n_pts), dtype=torch.int32, device=dev)
                row_base = torch.from_numpy(np.repeat(bases.astype(np.int32), counts)).to(dev)[:, None]
                stages = self._host_stages(walk_grasp_many(Ms, counts, n_pts, host_draw_stages(groups, self.chunk),
                                                           h_ids), h_ids, d_ids, row_base)
            ctx_engine = ctx.get_engine()
            ctx.set_engine(self.engine)         # the context (one per device) is shared: this predicter's engine, per call
            try:
                stale = self.engine >= 2 and ctx.fp16_overflow()
                for r0, r1, g0, g1 in stages:
                    forward(r0, r1, g0, g1, d_ids)
                overflow = self.engine >= 2 and ctx.fp16_overflow()
                for o in (live if overflow or stale else []):
                    r0, r1, (g0, g1) = int(offsets[o]), int(offsets[o + 1]), spans[o]
                    own = False
                    if overflow:
                        forward(r0, r1, g0, g1, d_ids)
                        own = ctx.fp16_overflow()
                    if own or (stale and o == live[0]):
                        print("GraspPredicter: activation beyond the fp16 range, re-running on engine 1 (wgmma bf16 "
                              "hi/lo x3)")
                        ctx.set_engine(1)
                        forward(r0, r1, g0, g1, d_ids)
                        ctx.set_engine(self.engine)
            finally:
                ctx.set_engine(ctx_engine)
        return d_probs, offsets

    def _host_stages(self, walk, h_ids, d_ids, row_base):
        """Runs ``walk`` (walk_grasp_many) on a worker thread and yields its stages as they are drawn, each copied to
        d_ids and rebased to the rows of the concatenated clouds (one add of row_base per stage)."""
        import queue
        import threading
        q = queue.Queue()

        def producer():
            try:
                for stage in walk:
                    q.put(stage)
                q.put(None)
            except Exception as e:   # surfaces in the consumer
                q.put(e)
        t = threading.Thread(target=producer, daemon=True)
        t.start()
        while (item := q.get()) is not None:
            if isinstance(item, Exception):
                t.join()
                raise item
            r0, r1 = item[0], item[1]
            d_ids[r0:r1].copy_(h_ids[r0:r1], non_blocking=True)
            d_ids[r0:r1].add_(row_base[r0:r1])
            yield item
        t.join()

    def predict_batch_many(self, datas, grasp_poses_list, ids=None, subsample=None):
        """``[self.predict_batch(d, g) for d, g in zip(datas, grasp_poses_list)]`` (with ``ids[o]`` for object o), bit
        for bit and with the same consumption of numpy's global generator: ``score_many`` and one copy to the host."""
        probs, off = self.score_many(datas, grasp_poses_list, ids=ids, subsample=subsample)
        host = probs.cpu().numpy()
        return [result_list(host[off[o]:off[o + 1]]) if off[o + 1] > off[o] else [] for o in range(len(off) - 1)]


def result_list(probs):
    """(B, n_out) host probabilities as the reference returns them (predicter.py:87-91): [label, confidence, probs]
    per candidate."""
    labels = probs.argmax(1)
    conf = probs[np.arange(len(probs)), labels]
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
        # "host": the reference's numpy draws, bit for bit (the transform's subset, then 2 x ransac_max_iter RANSAC
        # subsets drawn in C); "device": counter-based draws on the GPU from one numpy value, not the reference's
        # numbers, and no host walk of the generator
        self.subsample = "host"
        # predicter.py:162-163's locals: score the RANSAC hypotheses by the kd-tree evaluation (aligning.py:68-79) at
        # this voxel size, in either subsample mode; predict's 3 mm ratio between thresholds stays the residual one
        self.use_kdtree_for_eval = False
        self.kdtree_eval_resolution = 0.003

    THRESHOLDS = (0.003, 0.005)           # predicter.py:154, the RANSAC pass thresholds in the order predict tries them
    ERR_THRES = 0.003                     # predicter.py:163, the ratio predict compares between them
    MAX_DIMENSIONS = np.array([1.2, 1.2, 1.2])

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
        """predicter.py:135-203: (nocs_cloud, transform) or (None, None); numpy for numpy input, CUDA tensors for
        CUDA input.  Sets data_transformed, confidence_z, pred_bins and, with a pose, best_ratio and nocs_pose.
        ``ids`` (n_pts,) overrides the cloud subset; ``self.subsample`` picks the random numbers ("host" / "device")."""
        assert self.subsample in ("host", "device"), self.subsample
        self._kd_resolution()
        if self.subsample == "device":
            return self._predict_device(data, ids)
        if getattr(data["cloud_xyz"], "is_cuda", False):
            data = {k: (v.cpu().numpy() if hasattr(v, "is_cuda") else v) for k, v in data.items()}
            nocs, tf = self._predict_host(data, ids)
            return (None, None) if tf is None else self._on(self.model.device, nocs, tf)
        return self._predict_host(data, ids)

    def _on(self, dev, *arrays):
        import torch
        return tuple(torch.from_numpy(np.ascontiguousarray(a)).to(dev) for a in arrays)

    def _kd_resolution(self):
        """The kd-tree evaluation's voxel size when it is on, else None; ValueError for a bad size."""
        from .aligning import _resolution
        return _resolution(self.kdtree_eval_resolution) if self.use_kdtree_for_eval else None

    def _ransac(self, source, target, ids):
        from .aligning import ransac9d_pose
        return ransac9d_pose(source, target, ids, self.THRESHOLDS, max_scale=self.max_scale, min_scale=self.min_scale,
                             max_dimensions=self.MAX_DIMENSIONS, ratio_threshold=self.ERR_THRES,
                             kdtree_eval_resolution=self._kd_resolution())

    def _predict_host(self, data, ids):
        """The reference's numbers: the transform's subset from np.random.choice, then both thresholds' subsets in
        one C draw that continues numpy's stream where the reference's two loops would (aligning.py:91-97), one
        fused launch on them, and predict's post-processing in numpy on the two winners' T (predicter.py:152-172)."""
        nocs_cloud, _ = self.predict_nocs(data, ids=ids)
        ori_cloud = self.data_transformed["cloud_xyz_original"]
        symmetry_tf = np.eye(4)
        source = np.ascontiguousarray((symmetry_tf @ to_homo(nocs_cloud).T).T[:, :3], dtype=np.float64)
        target = np.ascontiguousarray(ori_cloud, dtype=np.float64)
        N, H = len(source), int(self.ransac_max_iter)
        if N < 4:
            raise ValueError("Cannot take a larger sample than population when 'replace=False'")   # as np.random.choice
        draw = _LegacyDraw()
        hyp = draw.draw(N, 4, len(self.THRESHOLDS) * H)
        draw.commit()
        dev = self.model.device
        res = self._ransac(*self._on(dev, source, target, hyp))
        best_ratio, best_transform = self._choose_host(res["record"].cpu().numpy(), source, target)
        if best_transform is None:
            return None, None
        self.best_ratio = best_ratio
        self.nocs_pose = best_transform.copy()
        nocs_cloud = (symmetry_tf @ to_homo(nocs_cloud).T).T[:, :3]
        return nocs_cloud, best_transform

    def _choose_host(self, record, source, target):
        """predict's choice between the thresholds in numpy (predicter.py:152-172) from a pose search's host record:
        (best_ratio, best_transform), best_transform None when no threshold gives a pose."""
        from .aligning import read_record
        found = read_record(record, len(self.THRESHOLDS))
        best_ratio = 0
        best_transform = None
        for t in range(len(self.THRESHOLDS)):
            if found["winner"][t] < 0:                                    # estimate9DTransform returned None
                continue
            transform = found["T"][t].copy()
            if np.linalg.det(transform[:3, :3]) < 0:
                continue
            transformed = (transform @ to_homo(source).T).T[:, :3]
            errs = np.linalg.norm(transformed - target, axis=1)
            ratio = np.sum(errs <= self.ERR_THRES) / len(errs)
            if ratio > best_ratio:
                best_ratio = ratio
                best_transform = transform.copy()
        return best_ratio, best_transform

    def device_transform(self, data, ids=None, seed=None):
        """transform() on the device in float64 for numpy or CUDA input: the z >= 0.1 mask, the subset (``ids``, else
        candidate 0 of cg_draw_ids_dev with ``seed``), the min/extent normalisation and the mean/std scaling.  With
        the same ids, 'input' equals transform()'s bit for bit.  Returns a dict of CUDA tensors ('cloud_xyz',
        'cloud_normal', 'cloud_xyz_original', 'keep_ids', 'input').  With CUDA input the masked point count is read
        on the host (one synchronisation): it sizes the draw."""
        import torch
        from . import _lib
        n_pts = int(self.cfg["n_pts"])
        ctx, xyz, nrm = _lib.inputs(data["cloud_xyz"], data["cloud_normal"], dtype=torch.float64, ctx=self.model.ctx)
        if getattr(data["cloud_xyz"], "is_cuda", False):
            keep_ids = torch.nonzero(data["cloud_xyz"][:, 2] >= 0.1).reshape(-1).to(xyz.device)   # in the input's dtype
        else:
            keep_ids = torch.from_numpy(np.nonzero(np.asarray(data["cloud_xyz"])[:, 2] >= 0.1)[0]).to(xyz.device)
        if ids is None:
            sub = self.model.draw_ids_dev(keep_ids.numel(), n_pts, 1, seed, first_candidate=0)[0].long()
        else:
            sub = torch.as_tensor(np.asarray(ids) if not hasattr(ids, "is_cuda") else ids).to(xyz.device).long()
        keep_ids = keep_ids[sub]
        x0, nr = xyz[keep_ids], nrm[keep_ids]
        mn = x0.amin(0)
        scale = (x0.amax(0) - mn).max()
        xn = (x0 - mn) / (scale + 1e-15)
        inp = torch.cat([xn, nr], 1)
        if "mean" in self.cfg:
            mean, std = self._on(xyz.device, self.cfg["mean"].reshape(1, -1), self.cfg["std"].reshape(1, -1))
            inp = (inp - mean) / (std + 1e-15)
        return {"cloud_xyz": xn, "cloud_normal": nr, "cloud_xyz_original": x0, "keep_ids": keep_ids, "input": inp}

    def _predict_device(self, data, ids):
        """Device mode: consumes ONE value of numpy's global generator (the seed, np.random.randint as
        GraspPredicter's device draw does).  Candidate 0 of cg_draw_ids_dev(seed) is the cloud subset, candidates
        1 .. H the first threshold's subsets and H+1 .. 2H the second's; the forward, the RANSAC and predict's
        choice between thresholds run on the device.  The host waits for the masked point count with CUDA input,
        and for the record (whether there is a pose, best_ratio) and, with numpy input, the copy of the results."""
        import torch
        from .aligning import read_record
        seed = int(np.random.randint(0, 2 ** 63 - 1, dtype=np.int64))
        cuda_in = getattr(data["cloud_xyz"], "is_cuda", False)
        H, n_thr = int(self.ransac_max_iter), len(self.THRESHOLDS)
        dt = self.device_transform(data, ids=ids, seed=seed)
        coords, conf_z, bins = self.model.nunocs_dev(dt["input"].to(torch.float32), int(self.cfg["ce_loss_bins"]))
        source = coords.to(torch.float64)
        hyp = self.model.draw_ids_dev(source.shape[0], 4, n_thr * H, seed, first_candidate=1)
        res = self._ransac(source, dt["cloud_xyz_original"], hyp)
        found = read_record(res["record"].cpu().numpy(), n_thr)
        host = (lambda t: t.cpu().numpy()) if not cuda_in else (lambda t: t)
        self.data_transformed = {k: host(v) for k, v in dt.items()}
        self.confidence_z, self.pred_bins = host(conf_z), host(bins)
        if found["chosen"] < 0:
            return None, None
        self.best_ratio = float(found["best_ratio"])
        pose = host(res["pose"].clone())
        self.nocs_pose = pose.copy() if not cuda_in else pose.clone()
        return host(source), pose

    def predict_many(self, datas, ids=None):
        """predict for a list of objects: ``[self.predict(d) for d in datas]`` (with ``ids[b]`` for object b), bit for
        bit, from the same state of numpy's global generator, which it leaves where the loop would; the attributes
        data_transformed, confidence_z, pred_bins, best_ratio and nocs_pose are left as the loop leaves them.
        ``datas`` are all numpy or all CUDA-tensor dicts with 'cloud_xyz' and 'cloud_normal' (M_b,3); they are not
        modified.  ``ids`` (optional) is a list of B subsets of n_pts indices into the masked cloud, or None entries.
        Returns one (nocs_cloud, pose) per object, (None, None) for an object with no pose.

        The random numbers are drawn first, in the loop's order (host mode: object b's cloud subset, then its
        2 x ransac_max_iter RANSAC subsets, in one walk of the generator; device mode: one seed per object), then
        the forward runs on all objects in one batched pass (cg_nunocs_forward_many_*) and the residual pose search
        in one launch over (object, threshold, hypothesis) (cg_ransac9d_pose_many_dev).  With use_kdtree_for_eval
        the pose search runs one object at a time after the batched forward, as each builds its own target index.

        The whole list is checked before any random number is drawn or any device work starts: a masked cloud that
        is empty (where predict's draw raises) gives predict's ValueError, and mixed or malformed inputs a
        ValueError.  So on error numpy's generator is left untouched, where the loop would have drawn for the
        objects before the failing one."""
        assert self.subsample in ("host", "device"), self.subsample
        self._kd_resolution()
        datas = list(datas)
        B = len(datas)
        ids = [None] * B if ids is None else [i if i is None or hasattr(i, "is_cuda") else np.asarray(i) for i in ids]
        cuda_in, counts = self._check_many(datas, ids)
        if B == 0:
            return []
        if self.subsample == "device":
            return self._predict_many_device(datas, ids, counts, cuda_in)
        if cuda_in:
            datas = [{k: (v.cpu().numpy() if hasattr(v, "is_cuda") else v) for k, v in d.items()} for d in datas]
            ids = [i if i is None or not hasattr(i, "is_cuda") else i.cpu().numpy() for i in ids]
            return [(None, None) if tf is None else self._on(self.model.device, nocs, tf)
                    for nocs, tf in self._predict_many_host(datas, ids, counts)]
        return self._predict_many_host(datas, ids, counts)

    def _check_many(self, datas, ids):
        """predict_many's checks, before any draw: (whether the inputs are CUDA tensors, masked point counts)."""
        import torch
        n_pts = int(self.cfg["n_pts"])
        if len(ids) != len(datas):
            raise ValueError(f"predict_many: {len(ids)} id subsets for {len(datas)} objects")
        if n_pts < 4:
            raise ValueError("Cannot take a larger sample than population when 'replace=False'")   # as predict
        kinds = set()
        for b, d in enumerate(datas):
            if not hasattr(d, "keys") or "cloud_xyz" not in d or "cloud_normal" not in d:
                raise ValueError(f"predict_many: object {b} is not a dict with 'cloud_xyz' and 'cloud_normal'")
            xyz, nrm = d["cloud_xyz"], d["cloud_normal"]
            for a in (xyz, nrm):
                kinds.add("cuda" if isinstance(a, torch.Tensor) and a.is_cuda else
                          "numpy" if isinstance(a, np.ndarray) else type(a).__name__)
            if len(kinds) > 1 or not kinds <= {"cuda", "numpy"}:
                raise ValueError(f"predict_many: the clouds must be all numpy arrays or all CUDA tensors, got "
                                 f"{sorted(kinds)}")
            if len(xyz.shape) != 2 or xyz.shape[1] != 3 or tuple(nrm.shape) != tuple(xyz.shape):
                raise ValueError(f"predict_many: object {b} has cloud_xyz {tuple(xyz.shape)} and cloud_normal "
                                 f"{tuple(nrm.shape)}; both must be (M,3)")
            if ids[b] is not None and tuple(ids[b].shape) != (n_pts,):
                raise ValueError(f"predict_many: ids[{b}] has shape {tuple(ids[b].shape)}, not ({n_pts},)")
        cuda_in = kinds == {"cuda"}
        if cuda_in:
            dev = self.model.device
            vals = [(d["cloud_xyz"][:, 2] >= 0.1).sum().to(dev) for d in datas]   # the mask in the input's dtype
            for i in ids:
                if i is not None:
                    i = torch.as_tensor(i).to(dev)
                    vals += [i.min(), i.max()]
            vals = torch.stack([v.to(torch.int64) for v in vals]).cpu().numpy()   # one synchronisation
            counts, lims = vals[:len(datas)], vals[len(datas):].reshape(-1, 2)
        else:
            counts = np.array([np.count_nonzero(np.asarray(d["cloud_xyz"])[:, 2] >= 0.1) for d in datas], np.int64)
            host_ids = [np.asarray(i.cpu() if hasattr(i, "is_cuda") else i) for i in ids if i is not None]
            lims = np.array([(i.min(), i.max()) for i in host_ids], np.int64).reshape(-1, 2)
        k = 0
        for b, M in enumerate(counts):
            if ids[b] is None:
                if M == 0:
                    raise ValueError("'a' cannot be empty unless no samples are taken")   # predict's np.random.choice
                continue
            if lims[k, 0] < 0 or lims[k, 1] >= M:
                raise ValueError(f"predict_many: ids[{b}] indexes outside the {M} points with z >= 0.1")
            k += 1
        return cuda_in, [int(M) for M in counts]

    def _predict_many_host(self, datas, ids, counts):
        """predict_many on numpy input in host mode: the draws in one walk, transform() per object, one forward, one
        pose search (or one per object with the kd-tree evaluation), one copy of the records, _choose_host."""
        import torch
        n_pts, H, B = int(self.cfg["n_pts"]), int(self.ransac_max_iter), len(datas)
        subs, hyp = draw_nunocs_many(counts, n_pts, len(self.THRESHOLDS) * H, given=ids)
        dts, xs = [], np.empty((B, n_pts, 6), dtype=np.float32)
        for b, data in enumerate(datas):
            d = dict(data)                                                  # predict_nocs, without writing to data
            d["cloud_nocs"] = np.zeros(d["cloud_xyz"].shape)
            d["cloud_rgb"] = np.zeros(d["cloud_xyz"].shape)
            dts.append(self.transform(copy.deepcopy(d), ids=subs[b] if ids[b] is None else ids[b]))
            xs[b] = np.ascontiguousarray(dts[b]["input"], dtype=np.float64).astype(np.float32)
        coords, conf_z, bins = self.model.nunocs_many_host(xs, int(self.cfg["ce_loss_bins"]))
        symmetry_tf = np.eye(4)
        source = [np.ascontiguousarray((symmetry_tf @ to_homo(coords[b]).T).T[:, :3], dtype=np.float64)
                  for b in range(B)]
        target = [np.ascontiguousarray(dt["cloud_xyz_original"], dtype=np.float64) for dt in dts]
        dev = self.model.device
        if self.use_kdtree_for_eval:
            recs = [self._ransac(*self._on(dev, source[b], target[b], hyp[b]))["record"] for b in range(B)]
            recs = torch.stack(recs)
        else:
            recs = self._ransac_many(*self._on(dev, np.stack(source), np.stack(target), hyp))
        recs = recs.cpu().numpy()
        out = []
        for b in range(B):                                                  # the attributes in the loop's order
            self.data_transformed, self.confidence_z, self.pred_bins = dts[b], conf_z[b], bins[b]
            best_ratio, best_transform = self._choose_host(recs[b], source[b], target[b])
            if best_transform is None:
                out.append((None, None))
                continue
            self.best_ratio = best_ratio
            self.nocs_pose = best_transform.copy()
            out.append((source[b], best_transform))
        return out

    def _ransac_many(self, source, target, ids):
        from .aligning import ransac9d_pose_many
        return ransac9d_pose_many(source, target, ids, self.THRESHOLDS, max_scale=self.max_scale,
                                  min_scale=self.min_scale, max_dimensions=self.MAX_DIMENSIONS,
                                  ratio_threshold=self.ERR_THRES)

    def _device_transform_many(self, datas, ids, seeds, counts):
        """device_transform for every object: (B,n_pts,*) CUDA tensors 'cloud_xyz', 'cloud_normal',
        'cloud_xyz_original', 'keep_ids' and 'input', row b bit for bit device_transform(datas[b], ids[b],
        seeds[b]).  The subsets are drawn per object (each has its own point count and seed); the gathers,
        normalisation and scaling run on all objects at once.  No synchronisation."""
        import torch
        from . import _lib
        n_pts, B = int(self.cfg["n_pts"]), len(datas)
        ctx = self.model.ctx
        xyz_all, nrm_all, keep, glob = [], [], [], []
        off = 0
        for b, d in enumerate(datas):
            _, xyz, nrm = _lib.inputs(d["cloud_xyz"], d["cloud_normal"], dtype=torch.float64, ctx=ctx)
            if getattr(d["cloud_xyz"], "is_cuda", False):
                k = torch.nonzero_static(d["cloud_xyz"][:, 2] >= 0.1, size=counts[b]).reshape(-1).to(xyz.device)
            else:
                k = torch.from_numpy(np.nonzero(np.asarray(d["cloud_xyz"])[:, 2] >= 0.1)[0]).to(xyz.device)
            if ids[b] is None:
                sub = self.model.draw_ids_dev(counts[b], n_pts, 1, seeds[b], first_candidate=0)[0].long()
            else:
                sub = torch.as_tensor(np.asarray(ids[b]) if not hasattr(ids[b], "is_cuda") else ids[b]).to(
                    xyz.device).long()
            keep.append(k[sub])
            glob.append(keep[-1] + off)
            off += xyz.shape[0]
            xyz_all.append(xyz)
            nrm_all.append(nrm)
        g = torch.cat(glob)
        x0 = torch.cat(xyz_all)[g].reshape(B, n_pts, 3)
        nr = torch.cat(nrm_all)[g].reshape(B, n_pts, 3)
        mn = x0.amin(1, keepdim=True)
        scale = (x0.amax(1, keepdim=True) - mn).amax(2, keepdim=True)
        xn = (x0 - mn) / (scale + 1e-15)
        inp = torch.cat([xn, nr], 2)
        if "mean" in self.cfg:
            mean, std = self._on(x0.device, self.cfg["mean"].reshape(1, 1, -1), self.cfg["std"].reshape(1, 1, -1))
            inp = (inp - mean) / (std + 1e-15)
        return {"cloud_xyz": xn, "cloud_normal": nr, "cloud_xyz_original": x0, "keep_ids": torch.stack(keep),
                "input": inp}

    def _predict_many_device(self, datas, ids, counts, cuda_in):
        """predict_many in device mode: B seeds (np.random.randint, in the loop's order), the batched transform and
        forward, each object's RANSAC subsets as candidates 1 .. 2H of cg_draw_ids_dev under its seed, one pose
        search, one copy of the records (and, with numpy input, one of the results)."""
        import torch
        from .aligning import REC_PER_THR
        n_thr, H, B = len(self.THRESHOLDS), int(self.ransac_max_iter), len(datas)
        seeds = [int(np.random.randint(0, 2 ** 63 - 1, dtype=np.int64)) for _ in range(B)]
        dt = self._device_transform_many(datas, ids, seeds, counts)
        coords, conf_z, bins = self.model.nunocs_many_dev(dt["input"].to(torch.float32), int(self.cfg["ce_loss_bins"]))
        source = coords.to(torch.float64)
        N = source.shape[1]
        hyp = torch.empty((B, n_thr * H, 4), dtype=torch.int32, device=source.device)
        for b in range(B):
            self.model.draw_ids_dev(N, 4, n_thr * H, seeds[b], first_candidate=1, out=hyp[b])
        if self.use_kdtree_for_eval:
            recs = torch.stack([self._ransac(source[b], dt["cloud_xyz_original"][b], hyp[b])["record"]
                                for b in range(B)])
        else:
            recs = self._ransac_many(source, dt["cloud_xyz_original"], hyp)
        rec_host = recs.cpu().numpy()
        if not cuda_in:
            dt = {k: v.cpu().numpy() for k, v in dt.items()}
            source, conf_z, bins = source.cpu().numpy(), conf_z.cpu().numpy(), bins.cpu().numpy()
        tail = n_thr * REC_PER_THR                                          # [chosen, pose (16), best_ratio]
        out = []
        for b in range(B):                                                  # the attributes in the loop's order
            self.data_transformed = {k: v[b] for k, v in dt.items()}
            self.confidence_z, self.pred_bins = conf_z[b], bins[b]
            if rec_host[b, tail] < 0:
                out.append((None, None))
                continue
            self.best_ratio = float(rec_host[b, tail + 17])
            pose = recs[b, tail + 1:tail + 17].reshape(4, 4).clone() if cuda_in else \
                rec_host[b, tail + 1:tail + 17].reshape(4, 4).copy()
            self.nocs_pose = pose.copy() if not cuda_in else pose.clone()
            out.append((source[b], pose))
        return out


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
            raise NotImplementedError("PointGroupPredictor: n_slice_per_side must be 1 (only whole frames are "
                                      "batched)")
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

    def predict_many(self, datas):
        """predict for a list of frames: ``[self.predict(d) for d in datas]`` bit for bit, numpy labels for numpy input
        and CUDA tensors for CUDA input, with self.xyz_shifted left as the loop leaves it (the last frame's).

        The front (device_front) runs per frame, so each frame keeps its own spatial shape.  The network then runs
        once over all frames: one batched spconv.index_many (its one synchronisation) and pyramid, one voxel mean, one
        U-Net forward and one offset head, with no synchronisation after the index.  The offsets are split by frame
        and pointgroup_labels runs per frame.

        The whole list is checked first: ValueError for an empty list, mixed numpy / CUDA frames, or a frame whose
        'cloud_xyz' and 'cloud_normal' are not both (M,3) with M >= 1; a frame without one of them gets predict's
        KeyError.  A rejected call does no device work and leaves self.xyz_shifted untouched."""
        import torch
        from . import spconv
        from .segment import MEANSHIFT_BANDWIDTH, pointgroup_labels
        datas = list(datas)
        cuda_in = self._check_many(datas)
        fronts = [self.device_front(d) for d in datas]
        level, p2v = spconv.index_many([f[1] for f in fronts], [f[3] for f in fronts])
        off = self.model.offsets(level, p2v, torch.cat([f[2] for f in fronts]))
        out, bw, start = [], MEANSHIFT_BANDWIDTH[self.class_name], 0
        for data, (xo, locs, _, _) in zip(datas, fronts):
            labels_all, xyz_shifted = pointgroup_labels(xo, off[start:start + len(locs)], data["cloud_xyz"], bw)
            start += len(locs)
            if not cuda_in:
                labels_all, xyz_shifted = labels_all.cpu().numpy(), xyz_shifted.cpu().numpy()
            out.append(labels_all)
        self.xyz_shifted = xyz_shifted
        return out

    @staticmethod
    def _check_many(datas):
        """predict_many's checks, before any device work: whether the frames are CUDA tensors."""
        import torch
        if not datas:
            raise ValueError("predict_many: no frames")
        kinds = set()
        for b, d in enumerate(datas):
            xyz, nrm = d["cloud_xyz"], d["cloud_normal"]                  # predict's KeyError for a missing array
            for a in (xyz, nrm):
                kinds.add("cuda" if isinstance(a, torch.Tensor) and a.is_cuda else
                          "numpy" if isinstance(a, np.ndarray) else type(a).__name__)
            if len(kinds) > 1 or not kinds <= {"cuda", "numpy"}:
                raise ValueError(f"predict_many: the frames must be all numpy arrays or all CUDA tensors, got "
                                 f"{sorted(kinds)}")
            if len(xyz.shape) != 2 or xyz.shape[1] != 3 or xyz.shape[0] == 0 or tuple(nrm.shape) != tuple(xyz.shape):
                raise ValueError(f"predict_many: frame {b} has cloud_xyz {tuple(xyz.shape)} and cloud_normal "
                                 f"{tuple(nrm.shape)}; both must be (M,3) with M >= 1")
        return kinds == {"cuda"}


def _float_dtype(a):
    """torch dtype of a float32 / float64 array or tensor (anything else is widened to float64)."""
    import torch
    name = str(a.dtype)
    return torch.float32 if name.endswith("float32") else torch.float64
