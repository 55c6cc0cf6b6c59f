"""Debug helper: compare engine 1 (wgmma, bf16 hi/lo x3) against engine 0 (fp32 SIMT) and the oracle."""
import sys, os, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from catgrasp_b200.net import PointNetCls
from catgrasp_b200.synthetic import make_state_dict
from oracle.pointnet_ref import pointnet_cls_forward
torch.cuda.set_device(0)
sd = make_state_dict("cls", 10, seed=0)
net = PointNetCls(sd, device=0)
for (B, N) in [(1, 128), (2, 300), (4, 1024), (64, 1024)]:
    rng = np.random.RandomState(B + N)
    x = rng.normal(0, 1, (B, N, 6)).astype(np.float32)
    ref = pointnet_cls_forward(sd, x)[0]
    out = {}
    for e in (0, 1, 2):
        net.ctx.set_engine(e)
        t = time.time()
        lg, pr = net.forward(x, return_probs=True)
        torch.cuda.synchronize()
        out[e] = (lg.cpu().numpy(), pr.cpu().numpy(), time.time() - t)
    print(f"B={B} N={N}: e0 vs ref dlogit {np.abs(out[0][0]-ref.numpy()).max():.2e}  "
          f"e1 vs ref dlogit {np.abs(out[1][0]-ref.numpy()).max():.2e} dprob {np.abs(out[1][1]-ref.softmax(1).numpy()).max():.2e}  "
          f"e2 vs ref dlogit {np.abs(out[2][0]-ref.numpy()).max():.2e} dprob {np.abs(out[2][1]-ref.softmax(1).numpy()).max():.2e}  "
          f"t0={out[0][2]*1e3:.1f}ms t1={out[1][2]*1e3:.1f}ms t2={out[2][2]*1e3:.1f}ms", flush=True)
