"""Times the iiwa14 IK feasibility test with CUDA events (DESIGN.md X5):
  * the IK kernel alone on 2^20 poses (counts only, and with the (Q,8,7) solutions written);
  * filterGraspPose's device route at 4096 x 12 pairs without IK, with the built-in IK pass, and the IK pass alone;
  * the host hook path (the reference's ikfast through oracle/_ref, when that build is present) on a subset.
Prints the card name and power limit read in the same run, then one line per measurement.

    python scripts/time_ik.py
"""
import _harness
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden"))

from catgrasp_b200 import my_cpp  # noqa: E402
from catgrasp_b200.ik import iiwa14_fk, iiwa14_ik  # noqa: E402
from catgrasp_b200.sdf import Sdf3D  # noqa: E402
from catgrasp_b200.synthetic import make_filter_case  # noqa: E402
from make_golden_mycpp import IK_LOWER, IK_UPPER, ik_frames  # noqa: E402


def timed(fn, reps=20):
    ts = _harness.synced_ms(fn, reps, 3)
    return float(np.median(ts)), float(np.min(ts))


def main():
    print("card:", _harness.card())
    rng = np.random.RandomState(0)
    Q = 1 << 20
    q = rng.uniform(-2.5, 2.5, (Q, 7))
    q[:, 2] = 0
    P = torch.from_numpy(iiwa14_fk(q).astype(np.float32)).cuda()
    med, mn = timed(lambda: iiwa14_ik(P, IK_UPPER, IK_LOWER))
    print(f"ik kernel, {Q} poses, counts only: median {med:.3f} ms (min {mn:.3f}) = {med * 1e6 / Q:.2f} ns/pose")
    med, mn = timed(lambda: iiwa14_ik(P, IK_UPPER, IK_LOWER, solutions=True))
    print(f"ik kernel, {Q} poses, with solutions: median {med:.3f} ms (min {mn:.3f})")

    G, S = 4096, 12
    p1, p2, poses, sym, nocs, c2n, g = make_filter_case(43, G, S, (1.0, 1.1, 0.9))
    so = Sdf3D(g["open"]["sdf"], g["open"]["origin"], g["open"]["res"], device=0)
    se = Sdf3D(g["enclosed"]["sdf"], g["enclosed"]["origin"], g["enclosed"]["res"], device=0)
    cam, ee = ik_frames()
    gp = torch.from_numpy(np.asarray(poses, np.float32)).cuda()
    args = (gp, sym, nocs, c2n, g["gripper_in_grasp"], True, True, so, p1, se, p2)
    ik = (cam, ee, IK_UPPER, IK_LOWER)
    base, _ = timed(lambda: my_cpp.filter_grasp_pose_raw(*args), reps=10)
    with_ik, _ = timed(lambda: my_cpp.filter_grasp_pose_raw(*args, ik=ik), reps=10)
    st, _, _ = my_cpp.filter_grasp_pose_raw(*args, ik=ik)
    st = st.cpu().numpy()
    print(f"filter {G}x{S} pairs: without IK {base:.3f} ms, with built-in IK {with_ik:.3f} ms "
          f"(IK pass ~{with_ik - base:.3f} ms); status counts {np.bincount(st, minlength=5).tolist()}")

    try:
        from oracle import mycpp_ref_ik
        have = mycpp_ref_ik.available()
    except Exception:      # noqa: BLE001
        have = False
    if have:
        n = 20000
        Ph = iiwa14_fk(q[:n]).astype(np.float32)
        t = time.perf_counter()
        for T in Ph:
            mycpp_ref_ik.ik_within_limits(T, IK_UPPER, IK_LOWER)
        dt = time.perf_counter() - t
        print(f"host ikfast (oracle build, one thread, via ctypes), {n} poses: {dt * 1e6 / n:.2f} us/pose")
    else:
        print("host ikfast: oracle/_ref not present, skipped")


if __name__ == "__main__":
    main()
