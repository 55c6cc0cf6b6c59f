"""Float64 reference of the folded PointNet encoder and heads, with a rigorous error bound -- ORACLE, test only.

It reads the packed weight blob of ``catgrasp_b200.weights.pack_blob`` (the exact fp32 weights the GPU gets), widens
it to float64 and runs each trunk and fully-connected layer.  Every value carries an absolute error bound ``e`` for
the GPU's result at the same place, propagated layer by layer:

    e_out = |W|^T e_in + u_layer * (|W|^T (|x| + e_in) + |b|)        (+ the fp16 subnormal term below)

ReLU and the max over points do not increase the error (|max a - max b| <= max |a - b|).  ``u_layer`` follows from
the arithmetic of the engine that runs the layer:

    fp32 FMA chain (engine 0 trunks, FMA FC kernels, every 6 -> 64 layer)   K * 2^-24
        any summation order of the K products and the bias makes at most K roundings
    bf16 hi/lo x3 (engines 1-3 L1 / L2, engine 1 L3, tensor-core FC)        max(2^-15, 3 * 2^-18 + K * 2^-24)
        x = hi + lo + r with |r| <= 2^-18 |x| for both operands, the dropped lo*lo term ~2^-18, fp32 accumulation
    engine 2 L3 (one fp16 term of W3, fp16 hi + lo activations)               2^-10
        2^-11 for the weight, 2^-21 for the activation split, accumulation K * 2^-24
    engine 3 L3 (fp16 x fp16)                                                 2^-10 + 2^-22 + K * 2^-24
    fp16 operands below 2^-14 are subnormal: each adds at most 2^-25 absolute, F16_ABS * (sum |x| + sum |W|)
    the xyz @ T3 product in the first trunk kernel                          3 * 2^-24
    the fused grasp-Q input (float64 transform narrowed to float32)         2^-24 |x|  (+ 2^-40 of the float64 terms)

Engines 2 and 3 fall back to engine 1 for a trunk whose folded W3 does not fit fp16 (``f16_ok``).  Values above the
fp16 range are outside these bounds on engines 2 and 3: there the kernels clamp and raise the overflow flag.

Layer order and the blob layout are those of csrc/cg_net.cu (layer_dims, pad64).
"""
import numpy as np
import torch

U32 = 2.0 ** -24
F16_ABS = 2.0 ** -25
FP16_MAX = 65504.0

ENCODER_LAYERS = [("S3_C1", 6, 64), ("S3_C2", 64, 128), ("S3_C3", 128, 1024), ("S3_F1", 1024, 512),
                  ("S3_F2", 512, 256), ("S3_F3", 256, 9), ("E_C1", 6, 64), ("SK_C1", 64, 64), ("SK_C2", 64, 128),
                  ("SK_C3", 128, 1024), ("SK_F1", 1024, 512), ("SK_F2", 512, 256), ("SK_F3", 256, 4096),
                  ("E_C2", 64, 128), ("E_C3", 128, 1024)]

# the three trunks: (6 -> 64, optional 64 -> 64, 64 -> 128, 128 -> 1024, ReLU after the last layer)
TRUNKS = {"A": ("S3_C1", None, "S3_C2", "S3_C3", True),      # STN3d
          "B": ("E_C1", "SK_C1", "SK_C2", "SK_C3", True),    # encoder conv1 + STNkd
          "C": ("E_C1", "T64", "E_C2", "E_C3", False)}       # encoder conv1, @T64, conv2, conv3 (BN, no ReLU)


def layer_dims(kind, n_out):
    d = [(n, k, c) for n, k, c in ENCODER_LAYERS]
    if kind == "cls":
        d += [("HEAD0", 1024, 512), ("HEAD1", 512, 256), ("HEAD2", 256, n_out), ("HEAD3", 0, 0), ("HEAD4", 0, 0)]
    else:
        d += [("HEAD0", 1024, 512), ("HEAD1", 64, 512), ("HEAD2", 512, 256), ("HEAD3", 256, 128),
              ("HEAD4", 128, n_out)]
    return d


def u_fp32(K):
    return K * U32


def u_bf16x3(K):
    return max(2.0 ** -15, 3 * 2.0 ** -18 + K * U32)


def u_l3(engine, K=128):
    """Unit roundoff of a trunk's 128 -> 1024 layer on ``engine`` (after the fp16 fallback has been resolved)."""
    if engine == 0:
        return u_fp32(K)
    if engine == 1:
        return u_bf16x3(K)
    if engine == 2:
        return 2.0 ** -10
    return 2.0 ** -10 + 2.0 ** -22 + K * U32


def key2f(k):
    """numpy twin of cg_key2f: order-preserving uint32 key -> float32."""
    k = np.asarray(k, dtype=np.uint32)
    b = np.where(k & np.uint32(0x80000000), k & np.uint32(0x7FFFFFFF), ~k).astype(np.uint32)
    return b.view(np.float32)


def f2key(f):
    """numpy twin of cg_f2key."""
    b = np.asarray(f, dtype=np.float32).view(np.uint32)
    return np.where(b & np.uint32(0x80000000), ~b, b | np.uint32(0x80000000)).astype(np.uint32)


def bound_ratio(got, ref, err, factor=2.0):
    """|got - ref| / (factor * err) elementwise; 0 where both are 0, inf where only the difference is."""
    got, ref, err = (np.asarray(a, dtype=np.float64) for a in (got, ref, err))
    d = np.abs(got - ref)
    lim = factor * err
    out = np.zeros(np.broadcast(d, lim).shape)
    pos = lim > 0
    np.divide(d, lim, out=out, where=pos)
    out[~pos & (d > 0)] = np.inf
    out[~np.isfinite(d)] = np.inf
    return out


def fused_input(xyz, nrm, poses, ids, mean=None, std=None):
    """The per-candidate input of the fused grasp-Q path (dataset_grasp.py:69-85) in float64, with the bound of the
    kernel's float32 narrowing.  xyz, nrm (M,3); poses (B,4,4); ids (B,N) or None (point n = cloud point n).
    Returns x (B,N,6) float64 and its error bound e (B,N,6)."""
    xyz, nrm, poses = (np.asarray(a, dtype=np.float64) for a in (xyz, nrm, poses))
    B = poses.shape[0]
    xs, es = [], []
    for b in range(B):
        sel = ids[b] if ids is not None else None
        p = xyz[sel] if sel is not None else xyz
        n = nrm[sel] if sel is not None else nrm
        inv = np.linalg.inv(poses[b])
        R, t = inv[:3, :3], inv[:3, 3]
        w = np.concatenate([p @ R.T + t, n @ R.T], axis=-1)
        mag = np.concatenate([np.abs(p) @ np.abs(R).T + np.abs(t), np.abs(n) @ np.abs(R).T], axis=-1)
        if mean is not None:
            sden = 1.0 / (np.asarray(std, np.float64).reshape(1, 6) + 1e-15)
            m = np.asarray(mean, np.float64).reshape(1, 6)
            w = (w - m) * sden
            mag = (mag + np.abs(m)) * sden
        xs.append(w)
        es.append(U32 * np.abs(w) + 2.0 ** -40 * mag)
    return np.stack(xs), np.stack(es)


class FoldedNet:
    """The folded network of one weight blob in float64 on ``device``."""

    def __init__(self, blob, kind, n_out, device="cpu"):
        self.kind, self.n_out = kind, int(n_out)
        self.device = torch.device(device)
        blob = np.asarray(blob, dtype=np.float32)
        self.W, self.b, self.w32max = {}, {}, {}
        off = 0
        for name, K, C in layer_dims(kind, n_out):
            nw = (K * C + 63) // 64 * 64
            nb = (C + 63) // 64 * 64
            if K:
                W = blob[off: off + K * C].reshape(K, C)
                self.W[name] = torch.from_numpy(W.astype(np.float64)).to(self.device)
                self.b[name] = torch.from_numpy(blob[off + nw: off + nw + C].astype(np.float64)).to(self.device)
                self.w32max[name] = float(np.abs(W).max())
            off += nw + nb
        assert off == blob.size, (off, blob.size)

    def f16_ok(self, trunk):
        """W3 of the trunk fits fp16, so engines 2 and 3 run it in fp16 (else they run the engine-1 kernel)."""
        return self.w32max[TRUNKS[trunk][3]] < FP16_MAX

    def trunk_engine(self, trunk, engine):
        return 1 if engine >= 2 and not self.f16_ok(trunk) else engine

    def _t(self, a):
        if a is None:
            return None
        if torch.is_tensor(a):
            return a.to(dtype=torch.float64, device=self.device)
        return torch.as_tensor(np.asarray(a), dtype=torch.float64, device=self.device)

    # ------------------------------------------------------------------------------------------------ layers
    @staticmethod
    def _lin(x, ex, W, b, u, f16=False):
        aW = W.abs()
        ax = x.abs() + ex
        y = x @ W
        mag = ax @ aW
        if b is not None:
            y = y + b
            mag = mag + b.abs()
        e = ex @ aW + u * mag
        if f16:
            e = e + F16_ABS * (ax.sum(-1, keepdim=True) + aW.sum(0))
        return y, e

    def fc(self, name, x, ex=None, relu=False, tc=False):
        """One fully-connected layer given its input rows x (M,K) and their bound: tc selects the bf16 hi/lo x3
        tensor-core unit roundoff, else the fp32 FMA one."""
        x = self._t(x)
        ex = torch.zeros_like(x) if ex is None else self._t(ex)
        W, b = self.W[name], self.b[name]
        K = W.shape[0]
        y, e = self._lin(x, ex, W, b, u_bf16x3(K) if tc else u_fp32(K))
        if relu:
            y = y.clamp_min(0.0)
        return y, e

    @staticmethod
    def fc_on_tc(engine, M, K, C):
        """cg_linear_launch runs a layer on tensor cores when all of these hold (cg_linear.cu): engine >= 1, at least
        64 rows, and the layer has a tensor-core image, which cg_linear_tc_image builds for K % 64 == 0 and C >= 64."""
        return engine >= 1 and M >= 64 and K % 64 == 0 and C >= 64

    # ------------------------------------------------------------------------------------------------ trunks
    def trunk_pre(self, which, x, ex=None, T3=None, eT3=None, T64=None, eT64=None, engine=1):
        """Per-point outputs of the trunk's 128 -> 1024 layer before bias, ReLU and max: z (B,N,1024) and its bound,
        plus the point feature after the optional 64 -> 64 stage (B,N,64) and its bound."""
        l0, l1, l2, l3, _ = TRUNKS[which]
        eng = self.trunk_engine(which, engine)
        x = self._t(x)
        ex = torch.zeros_like(x) if ex is None else self._t(ex)
        if T3 is not None:
            T = self._t(T3).reshape(-1, 3, 3)
            eT = torch.zeros_like(T) if eT3 is None else self._t(eT3).reshape(-1, 3, 3)
            p, ep = x[..., :3], ex[..., :3]
            ap = p.abs() + ep
            q = p @ T
            eq = ep @ T.abs() + ap @ eT + 3 * U32 * (ap @ T.abs())
            x = torch.cat([q, x[..., 3:]], -1)
            ex = torch.cat([eq, ex[..., 3:]], -1)
        h, e = self._lin(x, ex, self.W[l0], self.b[l0], u_fp32(6))
        h = h.clamp_min(0.0)
        u64 = u_fp32(64) if engine == 0 else u_bf16x3(64)
        if l1 == "T64":
            T = self._t(T64).reshape(-1, 64, 64)
            eT = torch.zeros_like(T) if eT64 is None else self._t(eT64).reshape(-1, 64, 64)
            ah = h.abs() + e
            h, e = h @ T, e @ T.abs() + ah @ eT + u64 * (ah @ T.abs())
        elif l1 is not None:
            h, e = self._lin(h, e, self.W[l1], self.b[l1], u64)
            h = h.clamp_min(0.0)
        pf, epf = h, e
        h, e = self._lin(h, e, self.W[l2], self.b[l2], u64)
        h = h.clamp_min(0.0)
        z, ez = self._lin(h, e, self.W[l3], None, u_l3(eng), f16=eng >= 2)
        # the kernel adds the bias after the max (one more fp32 rounding, inside the K * 2^-24 accumulation term)
        return z, ez, pf, epf

    def finish(self, which, zmax):
        """bias and ReLU after the max over points, as the kernel does."""
        y = zmax + self.b[TRUNKS[which][3]]
        return y.clamp_min(0.0) if TRUNKS[which][4] else y

    def trunk(self, which, x, ex=None, T3=None, eT3=None, T64=None, eT64=None, engine=1, want_pf=False,
              points_per_pass=1 << 17):
        """Max-pooled trunk output g (B,1024) and bound eg; with want_pf also the point feature (B,N,64) and its
        bound.  Candidates are processed in groups of at most ``points_per_pass`` points."""
        B, N = np.shape(x)[:2]
        step = max(1, points_per_pass // max(N, 1))
        g, eg, pf, epf = [], [], [], []
        for b0 in range(0, B, step):
            s = slice(b0, min(B, b0 + step))
            z, ez, p, ep = self.trunk_pre(which, x[s], None if ex is None else ex[s],
                                          None if T3 is None else T3[s], None if eT3 is None else eT3[s],
                                          None if T64 is None else T64[s], None if eT64 is None else eT64[s], engine)
            g.append(self.finish(which, z.amax(1)))
            eg.append(ez.amax(1))
            if want_pf:
                pf.append(p)
                epf.append(ep)
        out = {"g": torch.cat(g).cpu().numpy(), "eg": torch.cat(eg).cpu().numpy()}
        if want_pf:
            out["pf"], out["epf"] = torch.cat(pf).cpu().numpy(), torch.cat(epf).cpu().numpy()
        return out

    # ------------------------------------------------------------------------------------------------ FC chains
    # ``rows``: the row count of the GPU call (decides tensor cores vs FMA kernels); default the rows given here
    def stn_fc(self, which, g, eg=None, engine=1, rows=None):
        """The three FC layers after trunk A ('A' -> T3 (B,9)) or trunk B ('B' -> T64 (B,4096)), identity included."""
        names = ("S3_F1", "S3_F2", "S3_F3") if which == "A" else ("SK_F1", "SK_F2", "SK_F3")
        return self._chain(names, g, eg, engine, (True, True, False), rows)

    def cls_head(self, g, eg=None, engine=1, rows=None):
        return self._chain(("HEAD0", "HEAD1", "HEAD2"), g, eg, engine, (True, True, False), rows)

    def _chain(self, names, x, ex, engine, relus, rows=None):
        M = np.shape(x)[0] if rows is None else rows
        for name, relu in zip(names, relus):
            K, C = self.W[name].shape
            x, ex = self.fc(name, x, ex, relu=relu, tc=self.fc_on_tc(engine, M, K, C))
        return x.cpu().numpy(), ex.cpu().numpy()

    def seg_head(self, g, eg, pf, epf, engine=1):
        """PointNetSeg head (pointnet2.py:316-327) with the 1088 -> 512 conv split into its global half (per-cloud
        bias) and its point half, as cg_net.cu runs it.  Returns logits (B,N,n_out) and their bound."""
        B, N = np.shape(pf)[:2]
        P = B * N
        gb, egb = self.fc("HEAD0", g, eg, relu=False, tc=self.fc_on_tc(engine, B, 1024, 512))
        pf, epf = self._t(pf).reshape(P, 64), self._t(epf).reshape(P, 64)
        rep = torch.arange(P, device=self.device) // N
        y, e = self._lin(pf, epf, self.W["HEAD1"], None, u_bf16x3(64) if self.fc_on_tc(engine, P, 64, 512) else u_fp32(64))
        y = y + gb[rep]
        e = e + egb[rep] + U32 * (y.abs() + e + egb[rep])     # the per-cloud bias is one more fp32 addition
        y = y.clamp_min(0.0)
        for name, relu in (("HEAD2", True), ("HEAD3", True), ("HEAD4", False)):
            K, C = self.W[name].shape
            y, e = self.fc(name, y, e, relu=relu, tc=self.fc_on_tc(engine, P, K, C))
        return y.reshape(B, N, -1).cpu().numpy(), e.reshape(B, N, -1).cpu().numpy()

    # ------------------------------------------------------------------------------------------------ end to end
    def forward(self, x, ex=None, engine=1, rows=None):
        """Whole network in float64 with bounds.  x (B,N,6).  Returns a dict with the three trunk outputs (gA, gB,
        gC), T3, T64, the point feature (seg) and the logits, each with its bound (key prefixed 'e')."""
        out = {}
        A = self.trunk("A", x, ex, engine=engine)
        T3, eT3 = self.stn_fc("A", A["g"], A["eg"], engine, rows)
        Bt = self.trunk("B", x, ex, T3=T3, eT3=eT3, engine=engine)
        T64, eT64 = self.stn_fc("B", Bt["g"], Bt["eg"], engine, rows)
        C = self.trunk("C", x, ex, T3=T3, eT3=eT3, T64=T64, eT64=eT64, engine=engine, want_pf=self.kind == "seg")
        out.update(gA=A["g"], egA=A["eg"], gB=Bt["g"], egB=Bt["eg"], gC=C["g"], egC=C["eg"],
                   T3=T3, eT3=eT3, T64=T64, eT64=eT64)
        if self.kind == "cls":
            out["logits"], out["elogits"] = self.cls_head(C["g"], C["eg"], engine, rows)
        else:
            out["pf"], out["epf"] = C["pf"], C["epf"]
            out["logits"], out["elogits"] = self.seg_head(C["g"], C["eg"], C["pf"], C["epf"], engine)
        return out
