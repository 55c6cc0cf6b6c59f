"""Float64 sparse 3-D convolution by neighbour lookup, with a per-value error bound -- ORACLE, test only.

States the spconv 1.x semantics of csrc/cg_spconv.cu independently of it: levels from ``np.unique`` on the packed
site keys, neighbours by ``np.searchsorted``, and each convolution as one matrix product per kernel offset.  A dense
grid at PointGroup's 128^3 is too slow here; on small grids tests/test_spconv_ref.py holds this oracle to
``torch.nn.functional.conv3d`` / ``conv_transpose3d`` on zero-filled grids (spconv's own test contract).

Bound (the rule of encoder_ref.py): the device computes, per output, one fp32 FMA chain over n = K * Cin products,
then adds the bias and the residual.  With u = 2^-24, input bound ex and act(v) = max(v * s + t, 0):
    ea = |s| ex (1 + u) + u |s x + t|                 (BN prologue: one fmaf; ReLU does not increase it)
    ey = |W|^T ea + (n + 2) u (1 + 2^-20) (|W|^T (|a| + ea) + |b| + |res|) + eres
"""
import numpy as np

U32 = 2.0 ** -24
BITS = 21


def pack(c):
    c = np.asarray(c, dtype=np.int64)
    return (c[:, 0] << (2 * BITS)) | (c[:, 1] << BITS) | c[:, 2]


def unpack(k):
    k = np.asarray(k, dtype=np.int64)
    m = (1 << BITS) - 1
    return np.stack([(k >> (2 * BITS)) & m, (k >> BITS) & m, k & m], axis=1).astype(np.int32)


def neighbours(vox):
    """SubM k3 table (V,27): for k = 9 kx + 3 ky + kz the row of the site vox + (kx-1, ky-1, kz-1), or -1."""
    vox = np.asarray(vox, dtype=np.int64)
    keys = pack(vox)
    V = len(keys)
    nbr = np.full((V, 27), -1, dtype=np.int32)
    for k in range(27):
        q = vox + np.array([k // 9 - 1, k // 3 % 3 - 1, k % 3 - 1])
        ok = ((q >= 0) & (q < 1 << BITS)).all(1)
        qk = pack(np.where(ok[:, None], q, 0))
        pos = np.minimum(np.searchsorted(keys, qk), V - 1)
        hit = ok & (keys[pos] == qk)
        nbr[hit, k] = pos[hit]
    return nbr


def index(coords):
    """(vox (V,3) int32 in ascending key order, p2v (N,) int32, nbr (V,27) int32)."""
    keys, p2v = np.unique(pack(coords), return_inverse=True)
    vox = unpack(keys)
    return vox, p2v.astype(np.int32).reshape(-1), neighbours(vox)


def coarse_shape(shape):
    return tuple((s - 2) // 2 + 1 if s >= 2 else 0 for s in shape)


def down(vox, shape):
    """SparseConv3d(k2, s2) geometry: (coarse vox (P,3), coarse nbr (P,27), down (P,8), up (V,8), coarse shape)."""
    vox = np.asarray(vox, dtype=np.int64)
    cs = np.array(coarse_shape(shape))
    par = vox >> 1
    keep = (par < cs).all(1)
    keys = np.unique(pack(par[keep]))
    cvox = unpack(keys)
    parent = np.full(len(vox), -1, dtype=np.int64)
    parent[keep] = np.searchsorted(keys, pack(par[keep]))
    kc = (vox[:, 0] & 1) * 4 + (vox[:, 1] & 1) * 2 + (vox[:, 2] & 1)
    dn = np.full((len(keys), 8), -1, dtype=np.int32)
    up = np.full((len(vox), 8), -1, dtype=np.int32)
    c = np.nonzero(keep)[0]
    dn[parent[c], kc[c]] = c
    up[c, kc[c]] = parent[c]
    return cvox, neighbours(cvox), dn, up, tuple(int(s) for s in cs)


def conv(x, nbr, W, bn=None, bias=None, residual=None, ex=None, eres=None, rows=None):
    """out[r] = (sum_k W[k]^T act(x[nbr[r][k]]) + bias) + residual[r] in float64, and its bound (see the module
    docstring).  nbr None = the 1x1 convolution.  ``rows`` restricts the outputs to those rows.  Returns (y, ey)."""
    x = np.asarray(x, dtype=np.float64)
    Cin, Cout = W.shape[-2], W.shape[-1]
    W = np.asarray(W, dtype=np.float64).reshape(-1, Cin, Cout)
    K = W.shape[0]
    ex = np.zeros_like(x) if ex is None else np.asarray(ex, dtype=np.float64)
    if nbr is None:
        nbr = np.arange(len(x), dtype=np.int64)[:, None]
    nbr = np.asarray(nbr, dtype=np.int64)
    if rows is None:
        rows = np.arange(len(nbr))
    nbr = nbr[rows]
    if bn is None:
        a, ea = x, ex
    else:
        s, t = (np.asarray(v, dtype=np.float64) for v in bn)
        z = x * s + t
        a = np.maximum(z, 0.0)
        ea = np.abs(s) * ex * (1 + U32) + U32 * np.abs(z)
    y = np.zeros((len(rows), Cout))
    ey = np.zeros_like(y)
    mag = np.zeros_like(y)
    for k in range(K):
        m = nbr[:, k] >= 0
        src = nbr[m, k]
        Wk, Ak = W[k], np.abs(W[k])
        y[m] += a[src] @ Wk
        ey[m] += ea[src] @ Ak
        mag[m] += (np.abs(a[src]) + ea[src]) @ Ak
    if bias is not None:
        b = np.asarray(bias, dtype=np.float64)
        y += b
        mag += np.abs(b)
    if residual is not None:
        r = np.asarray(residual, dtype=np.float64)[rows]
        y += r
        mag += np.abs(r)
        if eres is not None:
            ey += np.asarray(eres, dtype=np.float64)[rows]
    ey += (K * Cin + 2) * U32 * (1 + 2.0 ** -20) * mag
    return y, ey


def dense_grid(vox, feats, shape):
    """Zero-filled (1, C, X, Y, Z) float64 grid with feats at the sites (for the dense comparison)."""
    g = np.zeros((1, feats.shape[1]) + tuple(shape))
    v = np.asarray(vox, dtype=np.int64)
    g[0][:, v[:, 0], v[:, 1], v[:, 2]] = np.asarray(feats, dtype=np.float64).T
    return g
