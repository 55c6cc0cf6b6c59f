"""X2 (SURVEY.md section 0, D2): how often does the gripper-SDF predicate agree with the reference's mesh-vs-occupied-voxel
predicate (FCL BVH x octomap OcTree, my_cpp/collision_manager.cpp:93-111) on the K2 workload?

FCL / octomap are not available (not in /root/reference, not installed, versions unpinned), so the reference side is the
float64 restatement of the SEMANTIC in oracle/fcl_semantic_ref.py (0.5 mm cubes at octomap keys vs posed triangles, 13-axis
SAT).  CPU only; run in the authoring container:

    python scripts/x2_agreement.py [--n 4096] [--procs 8]          -> JSON on stdout
"""
import argparse
import json
import multiprocessing as mp
import os
import sys
import time

import numpy as np

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)


def setup(n):
    """Mixed-verdict case (catgrasp_b200.synthetic.make_filter_case: an object crop + nearby background, poses from the
    cone parametrisation): on the K2 bench pile itself every candidate collides under all three predicates (checked:
    0 of 1024 accepted), which would make the agreement trivially 100 %."""
    from catgrasp_b200.synthetic import make_filter_case
    p1, p2, poses, sym, nocs_pose, c2n, g = make_filter_case(43, n, 1)
    return {"poses": poses, "open_pts": p1, "bg_pts": p2, "sym": sym, "nocs_pose": nocs_pose, "c2n": c2n}, g


def semantic_chunk(a):
    lo, hi, n = a
    from oracle import fcl_semantic_ref, filter_ref
    job, g = setup(n)
    none = np.zeros((0, 3))
    _, _, unshifted = filter_ref.filter_ref(job["poses"][lo:hi], job["sym"], job["nocs_pose"], job["c2n"], g["gripper_in_grasp"],
                                            False, False, 0, g["open"], none, g["enclosed"], none)
    out = np.zeros(hi - lo, bool)
    for i in range(hi - lo):
        gic = unshifted[i].astype(np.float64) @ g["gripper_in_grasp"]
        out[i] = (fcl_semantic_ref.mesh_hits_points(g["open"]["V"], g["open"]["F"], gic, job["open_pts"], 0.0005) or
                  fcl_semantic_ref.mesh_hits_points(g["enclosed"]["V"], g["enclosed"]["F"], gic, job["bg_pts"], 0.0005))
    return lo, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=4096)
    ap.add_argument("--procs", type=int, default=os.cpu_count())
    a = ap.parse_args()
    from catgrasp_b200.my_cpp import voxel_margin
    from oracle import filter_ref
    job, g = setup(a.n)
    t0 = time.time()
    verdict = {}
    for name, margin in (("sdf", 0.0), ("voxel", voxel_margin(0.0005))):
        st, _, _ = filter_ref.filter_ref(job["poses"], job["sym"], job["nocs_pose"], job["c2n"], g["gripper_in_grasp"], False, False,
                                         0, g["open"], job["open_pts"], g["enclosed"], job["bg_pts"], margin=margin)
        verdict[name] = st == 3
    step = max(1, a.n // (a.procs * 4))
    chunks = [(lo, min(a.n, lo + step), a.n) for lo in range(0, a.n, step)]
    sem = np.zeros(a.n, bool)
    with mp.get_context("spawn").Pool(a.procs) as pool:
        for lo, out in pool.imap_unordered(semantic_chunk, chunks):
            sem[lo:lo + len(out)] = out
    res = {"workload": "make_filter_case(seed 43): %d candidate poses against %d object + %d background points (no approach filter, no "
           "lateral adjustment), 0.5 mm voxels; on the K2 bench pile all candidates collide under every predicate" % (a.n, len(job["open_pts"]), len(job["bg_pts"])),
           "semantic_hits": int(sem.sum()), "seconds": round(time.time() - t0, 1)}
    for name in verdict:
        v = verdict[name]
        res[name] = {"agreement": float((v == sem).mean()), "predicate_only_hits": int((v & ~sem).sum()),
                     "semantic_only_hits": int((~v & sem).sum()), "hits": int(v.sum())}
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
