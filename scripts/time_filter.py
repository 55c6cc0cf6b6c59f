"""Times the collision filter alone on the bench workload (K2: 4096 candidates, 20k-pt scene)."""
import _harness
import types
import numpy as np, torch
import bench
from catgrasp_b200 import my_cpp
from catgrasp_b200.sdf import Sdf3D
from catgrasp_b200.synthetic import make_gripper_proxy


def main():
    print("card:", _harness.card())
    args = types.SimpleNamespace(n_pts=1024, nunocs_pts=8192, gpus=1)
    wl = bench.make_scene_job("K2", 0, 0, 4096, 4096, args, 0)
    g = make_gripper_proxy()
    so = Sdf3D(g["open"]["sdf"], g["open"]["origin"], g["open"]["res"])
    se = Sdf3D(g["enclosed"]["sdf"], g["enclosed"]["origin"], g["enclosed"]["res"])
    dev = torch.device("cuda", 0)
    d_pose32 = torch.from_numpy(wl["poses"]).to(dev).float().contiguous()
    d_open = torch.from_numpy(wl["open_pts"]).to(dev)
    d_bg = torch.from_numpy(wl["bg_pts"]).to(dev)
    eye = np.eye(4)
    run = lambda: my_cpp.filter_grasp_pose_raw(d_pose32, eye[None], eye, eye, g["gripper_in_grasp"], True, True, so, d_open, se, d_bg)
    st, off, _p = run()                  # the verdicts; the first of five warm-up calls
    ms = float(np.mean(_harness.queued_ms(run, 50, 4)))

    def timed(bg, op, tag):
        r = lambda: my_cpp.filter_grasp_pose_raw(d_pose32, eye[None], eye, eye, g["gripper_in_grasp"], True, True, so, op, se, bg)
        s2, o2, _q = r()                 # the first of three warm-up calls
        t = float(np.mean(_harness.queued_ms(r, 50, 2)))
        print(f"{tag}: {t * 1e3:.1f} us; same verdicts {bool((s2 == st).all().item() and (o2 == off).all().item())}")

    c = d_open.double().mean(0)
    for name, pts in (("bg", d_bg),):
        d2 = ((pts.double() - c) ** 2).sum(1)
        timed(pts[torch.argsort(d2)].contiguous(), d_open, "bg sorted by distance to the object centroid")
        timed(pts[torch.argsort(d2, descending=True)].contiguous(), d_open, "bg sorted far-first (worst case)")
        timed(pts[torch.randperm(pts.shape[0], device=dev)].contiguous(), d_open, "bg shuffled")
        # raster order of an occupancy image: rows of constant y (1 mm bins), x ascending inside a row
        key = torch.floor(pts[:, 1].double() * 1000.0) * 1e6 + pts[:, 0].double()
        timed(pts[torch.argsort(key)].contiguous(), d_open, "bg in raster order (y rows, x ascending)")
    print(f"filter: {ms * 1e3:.1f} us per call; accepted {(st == 0).sum().item()}, offsets {np.bincount(off.cpu().numpy().astype(np.int64) + 1).tolist()}, checksum {int(st.sum().item())}")


if __name__ == "__main__":
    main()
