"""CPU: GraspPredicter.predict_batch_many's host logic, which needs no device.

- walk_grasp_many (the host-mode subsets of several objects in one walk of numpy's generator) equals a loop of
  draw_subsample_ids_numpy, id for id and in the generator's state afterwards: objects with M < n_pts, M == n_pts and
  M > n_pts, objects with no candidates, and stages cut at every chunk edge (1023 / 1024 / 1025).
- graspq_fc_groups gives the launch cuts of a loop of one-object calls: ``chunk`` candidates per launch in host mode,
  the whole list in device and given-ids modes, each launch cut at GRASPQ_CHUNK_B as cg_graspq_forward_dev cuts it.
- A rejected list, or a rejected one-object score call, leaves numpy's generator untouched, in both subsample modes
  and with given ids.
- The Python constants match the header's, and the codegen of the two kernels the batched path extends.
"""
import contextlib
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from catgrasp_b200 import build
from catgrasp_b200.predicter import (GRASPQ_CHUNK_B, GraspPredicter, draw_subsample_ids_numpy, graspq_fc_groups,
                                     host_draw_stages, walk_grasp_many)


def _state():
    s = np.random.get_state()
    return s[0], s[1].copy(), s[2], s[3], s[4]


def _same(a, b):
    return a[0] == b[0] and np.array_equal(a[1], b[1]) and a[2:] == b[2:]


def _loop_ids(Ms, counts, n_pts):
    parts = [draw_subsample_ids_numpy(M, n_pts, c) for M, c in zip(Ms, counts) if c > 0]
    return np.concatenate(parts) if parts else np.empty((0, n_pts), np.int32)


@pytest.mark.parametrize("chunk", [1023, 1024, 1025, 5])
def test_walk_equals_loop_of_numpy_choice(chunk):
    n_pts = 16
    Ms = [40, 16, 9, 300, 16, 25, 1]                  # above, at and below n_pts (replace = M < n_pts)
    counts = [3, 0, 1024, 1, 1025, 0, 1023]
    groups, _ = graspq_fc_groups(counts, chunk)
    np.random.seed(5)
    want = _loop_ids(Ms, counts, n_pts)
    after = _state()
    np.random.seed(5)
    out = np.full((sum(counts), n_pts), -1, np.int32)
    stages = host_draw_stages(groups, chunk)
    seen = list(walk_grasp_many(Ms, counts, n_pts, stages, out))
    assert seen == stages
    assert np.array_equal(out, want)
    assert _same(after, _state())


def test_walk_over_objects_with_no_candidates_draws_nothing():
    np.random.seed(3)
    before = _state()
    assert list(walk_grasp_many([5, 7], [0, 0], 4, host_draw_stages(np.zeros(0, np.int32), 1024),
                                np.empty((0, 4), np.int32))) == []
    assert _same(before, _state())


def test_stages_pack_whole_groups():
    assert host_draw_stages([1, 7, 1024, 1, 1023, 1], 1024) == [(0, 8, 0, 2), (8, 1032, 2, 3), (1032, 2056, 3, 5),
                                                                (2056, 2057, 5, 6)]
    assert host_draw_stages([2000], 1024) == [(0, 2000, 0, 1)]
    assert host_draw_stages([], 1024) == []


class _Net:
    """A stand-in network: the calls below return before any launch."""
    device, n_out, ctx = torch.device("cpu"), 2, None


def _predicter(n_pts=8, chunk=1024, subsample="host", net=None):
    p = object.__new__(GraspPredicter)
    p.cfg = {"n_pts": n_pts}
    p.subsample, p.chunk, p._pin, p.engine = subsample, chunk, None, 3
    p.model = net
    p._pinned_ids = lambda B, n: torch.empty((B, n), dtype=torch.int32)
    return p


def _obj(M, seed, z=0.7):
    rng = np.random.RandomState(seed)
    xyz = rng.uniform(-0.02, 0.02, (M, 3))
    xyz[:, 2] += z
    return {"cloud_xyz": xyz, "cloud_normal": rng.normal(size=(M, 3))}


BIG = 2 * GRASPQ_CHUNK_B + 5
# per (mode, chunk), the FC row groups of the counts that are not one group of themselves
CUTS = {("host", 1024): {1025: [1024, 1], BIG: [1024] * 32 + [5]},
        ("host", 3): {7: [3, 3, 1], 8: [3, 3, 2], 9: [3, 3, 3], 63: [3] * 21, 64: [3] * 21 + [1], 65: [3] * 21 + [2],
                      1023: [3] * 341, 1024: [3] * 341 + [1], 1025: [3] * 341 + [2], BIG: [3] * 10924 + [1]},
        ("host", 20000): {BIG: [GRASPQ_CHUNK_B, 20000 - GRASPQ_CHUNK_B, BIG - 20000]},
        ("device", 1024): {BIG: [GRASPQ_CHUNK_B, GRASPQ_CHUNK_B, 5]},
        ("given", 1024): {BIG: [GRASPQ_CHUNK_B, GRASPQ_CHUNK_B, 5]}}


@pytest.mark.parametrize("mode, chunk", [("host", 1024), ("host", 3), ("host", 20000), ("device", 1024),
                                         ("given", 1024)])
def test_fc_groups_follow_the_launch_rule(mode, chunk):
    """A one-object call launches ``chunk`` candidates at a time in host mode and its whole list in device and
    given-ids modes, and cg_graspq_forward_dev runs each launch in passes of at most GRASPQ_CHUNK_B candidates."""
    counts = [0, 1, 7, 8, 9, 63, 64, 65, 1023, 1024, 1025, BIG]
    groups, spans = graspq_fc_groups(counts, chunk if mode == "host" else None)
    for o, B in enumerate(counts):
        want = CUTS[mode, chunk].get(B, [B] if B else [])
        assert list(groups[spans[o, 0]:spans[o, 1]]) == want, (o, B)
    assert spans[0, 0] == spans[0, 1] and groups.sum() == sum(counts)


def _rejects(p, datas, grasps, match, ids=None, one=False):
    """predict_batch_many(datas, grasps) raises, or with ``one`` score on the one object, and draws nothing."""
    np.random.seed(11)
    before = _state()
    with pytest.raises(ValueError, match=match):
        if one:
            p.score(datas[0], grasps[0], ids=None if ids is None else ids[0])
        else:
            p.predict_batch_many(datas, grasps, ids=ids)
    assert _same(before, _state())


@pytest.mark.parametrize("mode", ["host", "device"])
def test_rejected_list_leaves_the_generator_untouched(mode):
    p = _predicter(subsample=mode)
    good, g2 = _obj(30, 1), [np.eye(4)] * 2
    far = _obj(20, 2, z=0.05)                                # every point below z = 0.1
    _rejects(p, [good, good, far], [g2, g2, g2], "cannot be empty unless no samples are taken")
    _rejects(p, [good, good], [g2], "pose lists")
    _rejects(p, [good, good], [g2, [np.eye(3)]], "not 4x4")
    _rejects(p, [good, {"cloud_xyz": np.zeros((4, 3))}], [g2, g2], "is not a dict")
    _rejects(p, [good, {"cloud_xyz": np.ones((4, 3)), "cloud_normal": np.ones((5, 3))}], [g2, g2], "must be")
    _rejects(p, [good, good], [g2, g2], "id arrays", ids=[np.zeros((2, 8), np.int32)])
    _rejects(p, [good, good], [g2, g2], "has shape", ids=[np.zeros((2, 8), np.int32), np.zeros((2, 7), np.int32)])
    _rejects(p, [good, good], [g2, g2], "indexes outside",
             ids=[np.zeros((2, 8), np.int32), np.full((2, 8), 30, np.int32)])
    _rejects(p, [far], [g2], "cannot be empty unless no samples are taken", one=True)
    _rejects(p, [good], [g2], "has shape", ids=[np.zeros((2, 7), np.int32)], one=True)
    _rejects(p, [good], [g2], "indexes outside", ids=[np.full((2, 8), 30, np.int32)], one=True)


def test_objects_without_candidates_are_not_checked(monkeypatch):
    """predict_batch returns [] for an empty pose list before it looks at the data: so does the batched call."""
    monkeypatch.setattr(torch.cuda, "device", lambda d: contextlib.nullcontext())
    p = _predicter(net=_Net())
    np.random.seed(2)
    before = _state()
    assert p.predict_batch_many([_obj(20, 2, z=0.05), None], [[], []]) == [[], []]
    assert _same(before, _state())


def test_chunk_constant_matches_the_header():
    hdr = open(os.path.join(build.HERE, "..", "include", "catgrasp_b200.h")).read()
    assert int(re.search(r"#define CG_GRASPQ_CHUNK_B (\d+)", hdr).group(1)) == GRASPQ_CHUNK_B


NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")


def _ptxas(src):
    flags = [f for f in build.NVCC_FLAGS if f != "-DCG_EXPERIMENTS"]
    r = subprocess.run([NVCC] + flags + ["-Xptxas", "-v", "-c", os.path.join(build.CSRC, src), "-o", os.devnull],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout
    out = {}
    for m in re.finditer(r"Function properties for (\S+)\s*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                         r"(\d+) bytes spill loads\s*\n.*?Used (\d+) registers", r.stdout):
        out[m.group(1)] = tuple(int(v) for v in m.groups()[1:])
    return out


@pytest.mark.skipif(shutil.which(NVCC) is None, reason="nvcc not available")
def test_grouped_kernels_keep_registers_and_the_trunk_its_register_counts():
    """The few-row FC kernel with its group table and the draw kernel with its object table keep a 0-byte stack and
    no spills.  The batched path leaves the trunk kernels as they were: with CUDA 12.9 ptxas gives them the register
    counts they had before it (168 / 162 / 164 for the tensor-core engines 1-3, 185 for the SIMT engine)."""
    for src, name in (("cg_linear.cu", "18linear_rows_kernel"), ("cg_draw.cu", "15draw_ids_kernel")):
        rec = {k: v for k, v in _ptxas(src).items() if name in k}
        assert len(rec) == 1, rec
        assert list(rec.values())[0][:3] == (0, 0, 0), rec
    ver = subprocess.run([NVCC, "--version"], stdout=subprocess.PIPE, text=True).stdout
    if "release 12.9" not in ver:
        pytest.skip("the trunk's register counts are recorded for CUDA 12.9")
    regs = {k: v[3] for k, v in {**_ptxas("cg_trunk_tc.cu"), **_ptxas("cg_trunk_simt.cu")}.items()}
    want = {"trunk_tc_kernelILi1EE": 168, "trunk_tc_kernelILi2EE": 162, "trunk_tc_kernelILi3EE": 164,
            "trunk_simt_kernel": 185}
    for key, n in want.items():
        hit = [v for k, v in regs.items() if key in k]
        assert hit == [n], (key, regs)
