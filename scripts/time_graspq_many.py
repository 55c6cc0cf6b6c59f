"""GraspPredicter.predict_batch_many against the loop of predict_batch calls it replaces, in both subsample modes
(synthetic 'cls' weights, n_pts 2048, engine 3).  The two forms run alternately, each from the same numpy seed, and
their results are compared bit for bit.  Workloads:

  pick16 -- 16 objects of a synthetic pile with 1 to 64 grasps each (seeded counts);
  pile   -- the objects of the time_pick.py frame (16 objects rendered with the reference camera), 1 to 64 grasps each;
  K4     -- 8 scenes x 4096 candidates (the shape of bench.py's K4 per scene).

    python scripts/time_graspq_many.py [--reps 5] [--n-pts 2048] [--only pick16,pile,K4]
"""
import _harness
import argparse
import tempfile

import numpy as np

from catgrasp_b200 import cloud, synthetic
from catgrasp_b200.predicter import GraspPredicter

K = _harness.REFERENCE_K


def _objects(clouds, counts, seed):
    datas, grasps = [], []
    for o, (ob, B) in enumerate(zip(clouds, counts)):
        datas.append(ob)
        grasps.append(list(synthetic.make_candidates(ob["cloud_xyz"], ob["cloud_normal"], int(B), seed=seed + o)))
    return datas, grasps


def _pile_objects(n_points, n_objects, seed):
    scene = synthetic.make_pile(n_points, n_objects=n_objects, seed=seed)
    return [{"cloud_xyz": scene["cloud_xyz"][scene["object_id"] == k],
             "cloud_normal": scene["cloud_normal"][scene["object_id"] == k]} for k in range(n_objects)]


def _frame_objects():
    depth, ids = synthetic.render_depth(K, *_harness.REFERENCE_HW, n_objects=16, seed=1)
    xyz = cloud.depth2xyzmap(depth, K)
    lab = ids[ids >= 0]
    pts = xyz[ids >= 0].reshape(-1, 3)
    out = []
    for k in np.unique(lab):
        ob = pts[lab == k]
        out.append({"cloud_xyz": ob, "cloud_normal": cloud.estimate_normals(ob, 0.002, 30)})
    return out


def _same(a, b):
    return len(a) == len(b) and all(
        len(x) == len(y) and all(u[0] == v[0] and u[2].tobytes() == v[2].tobytes() for u, v in zip(x, y))
        for x, y in zip(a, b))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--n-pts", type=int, default=2048)
    ap.add_argument("--only", default="pick16,pile,K4")
    a = ap.parse_args()
    print("card:", _harness.card())
    tmp = tempfile.mkdtemp()
    gp = GraspPredicter("nut", artifact_dir=synthetic.write_artifacts(f"{tmp}/cls", "cls", a.n_pts, seed=3), device=0,
                        engine=3)
    rng = np.random.RandomState(0)
    work = {}
    if "pick16" in a.only:
        work["pick16"] = _objects(_pile_objects(16000, 16, 2), rng.randint(1, 65, 16), 100)
    if "pile" in a.only:
        frame = _frame_objects()
        work["pile"] = _objects(frame, rng.randint(1, 65, len(frame)), 200)
    if "K4" in a.only:
        work["K4"] = _objects(_pile_objects(20000, 8, 3), [4096] * 8, 300)
    for name, (datas, grasps) in work.items():
        sizes = [len(g) for g in grasps]
        print(f"{name}: {len(datas)} objects of {min(len(d['cloud_xyz']) for d in datas)} to "
              f"{max(len(d['cloud_xyz']) for d in datas)} points, {sum(sizes)} grasps ({min(sizes)} to {max(sizes)} "
              f"per object), n_pts {a.n_pts}, engine {gp.engine}")
        forms = {"loop": lambda: [gp.predict_batch(d, g) for d, g in zip(datas, grasps)],
                 "many": lambda: gp.predict_batch_many(datas, grasps)}
        for mode in ("host", "device"):
            gp.subsample = mode
            times, out = {f: [] for f in forms}, {}

            def run(f):
                np.random.seed(0)
                out[f] = forms[f]()
            for f in forms:                                   # warm-up
                run(f)
            for _ in range(a.reps):
                for f in forms:
                    times[f] += _harness.wall_ms(lambda: run(f), 1, 0)
            print(f"  {mode}: many == loop bit for bit: {_same(out['loop'], out['many'])}")
            for f in forms:
                print(f"    {name} {mode} {f:5s} {_harness.summary(times[f])}")
            print(f"    {name} {mode} loop / many (medians) {np.median(times['loop']) / np.median(times['many']):.2f}")


if __name__ == "__main__":
    main()
