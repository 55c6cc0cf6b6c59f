"""Checkpoint loading, BatchNorm folding and weight-blob packing.

Mirrors the loader contract of the reference (Utils.py:135-148 ``load_model``:
``map_location=cpu``, unwrap ``'state_dict'``, strip ``module.``) and produces
the fp32 blob consumed by ``cg_net_create`` (catgrasp_b200/csrc/cg_net.cu).

Folding (eval-mode BatchNorm1d, eps=1e-5, done in float64 then narrowed):
    y = gamma * (W x + b - mean) / sqrt(var + eps) + beta
      = (gamma/s) W x + (gamma/s) (b - mean) + beta ,  s = sqrt(var + eps)
Every layer is stored transposed, ``Wt[K][C_out]`` (k-major rows), followed by
its bias; each array is zero-padded to a multiple of 64 floats.
"""
from collections import OrderedDict

import numpy as np

BN_EPS = 1e-5  # torch.nn.BatchNorm1d default, pointnet2.py:164-168

# (blob slot, conv/linear prefix, bn prefix or None) -- order == cg_layer_id in csrc/cg_net.cuh
_ENCODER = [
    ("S3_C1", "feat.stn.conv1", "feat.stn.bn1"),
    ("S3_C2", "feat.stn.conv2", "feat.stn.bn2"),
    ("S3_C3", "feat.stn.conv3", "feat.stn.bn3"),
    ("S3_F1", "feat.stn.fc1", "feat.stn.bn4"),
    ("S3_F2", "feat.stn.fc2", "feat.stn.bn5"),
    ("S3_F3", "feat.stn.fc3", None),
    ("E_C1", "feat.conv1", "feat.bn1"),
    ("SK_C1", "feat.fstn.conv1", "feat.fstn.bn1"),
    ("SK_C2", "feat.fstn.conv2", "feat.fstn.bn2"),
    ("SK_C3", "feat.fstn.conv3", "feat.fstn.bn3"),
    ("SK_F1", "feat.fstn.fc1", "feat.fstn.bn4"),
    ("SK_F2", "feat.fstn.fc2", "feat.fstn.bn5"),
    ("SK_F3", "feat.fstn.fc3", None),
    ("E_C2", "feat.conv2", "feat.bn2"),
    ("E_C3", "feat.conv3", "feat.bn3"),
]
BLOB_ORDER = [s for s, _, _ in _ENCODER] + ["HEAD0", "HEAD1", "HEAD2", "HEAD3", "HEAD4"]


def strip_module_prefix(state_dict):
    """Utils.py:141-145: checkpoints saved from nn.DataParallel carry 'module.' prefixes."""
    if "state_dict" in state_dict:
        state_dict = state_dict["state_dict"]
    out = OrderedDict()
    for k, v in state_dict.items():
        out[k.replace("module.", "")] = v
    if len(out) == 0:
        raise RuntimeError("empty checkpoint")
    return out


def load_checkpoint(ckpt_path):
    """torch.load(..., map_location='cpu') + unwrap + strip, like Utils.py:135-145."""
    import torch
    sd = torch.load(ckpt_path, map_location=torch.device("cpu"), weights_only=False)
    return strip_module_prefix(sd)


def _np64(t):
    if hasattr(t, "detach"):
        t = t.detach().cpu().numpy()
    return np.asarray(t, dtype=np.float64)


def _fold(sd, lin, bn):
    """Return (Wt [K][C], b [C]) float64 with the BatchNorm folded in."""
    W = _np64(sd[lin + ".weight"])
    if W.ndim == 3:  # Conv1d(k=1): (C_out, C_in, 1)
        W = W[:, :, 0]
    b = _np64(sd[lin + ".bias"])
    if bn is not None:
        g = _np64(sd[bn + ".weight"])
        beta = _np64(sd[bn + ".bias"])
        mu = _np64(sd[bn + ".running_mean"])
        var = _np64(sd[bn + ".running_var"])
        s = g / np.sqrt(var + BN_EPS)
        W = W * s[:, None]
        b = (b - mu) * s + beta
    return W.T.copy(), b


def fold_mlp(state_dict, nlayers):
    """The fp32 (Wt [K][C], b [C]) of every layer of a PointNet++ shared-MLP stack (upstream layout mlp_convs.{i} +
    mlp_bns.{i}, Conv1d or Conv2d 1x1), BatchNorm folded: the exact weights ``cg_mlp_create`` receives."""
    sd = {k.replace("module.", ""): v for k, v in state_dict.items()}
    Wts, bs = [], []
    for i in range(nlayers):
        w = {k: _np64(v) for k, v in sd.items() if k.startswith(f"mlp_convs.{i}.") or k.startswith(f"mlp_bns.{i}.")}
        w[f"mlp_convs.{i}.weight"] = w[f"mlp_convs.{i}.weight"].reshape(w[f"mlp_convs.{i}.weight"].shape[0], -1, 1)
        Wt, b = _fold(w, f"mlp_convs.{i}", f"mlp_bns.{i}")
        Wts.append(np.ascontiguousarray(Wt, dtype=np.float32))
        bs.append(np.ascontiguousarray(b, dtype=np.float32))
    return Wts, bs


def _pad64(a):
    a = np.ascontiguousarray(a, dtype=np.float32).reshape(-1)
    n = (a.size + 63) // 64 * 64
    out = np.zeros(n, dtype=np.float32)
    out[: a.size] = a
    return out


def expected_keys(kind):
    keys = []
    heads = ([("fc1", "bn1"), ("fc2", "bn2"), ("fc3", None)] if kind == "cls" else
             [("conv1", "bn1"), ("conv2", "bn2"), ("conv3", "bn3"), ("conv4", None)])
    for _, lin, bn in _ENCODER + [("", l, b) for l, b in heads]:
        keys += [lin + ".weight", lin + ".bias"]
        if bn:
            keys += [bn + s for s in (".weight", ".bias", ".running_mean", ".running_var")]
    return keys


def check_state_dict(sd, kind):
    """Strict key check in the spirit of load_state_dict(strict=True), Utils.py:148."""
    need = set(expected_keys(kind))
    have = set(k for k in sd.keys() if not k.endswith("num_batches_tracked"))
    missing, extra = sorted(need - have), sorted(have - need)
    if missing or extra:
        raise RuntimeError(f"checkpoint does not match PointNet{'Cls' if kind == 'cls' else 'Seg'}: "
                           f"missing={missing[:8]} unexpected={extra[:8]}")


def pack_blob(sd, kind):
    """Fold + pack a PointNetCls ('cls') or PointNetSeg ('seg') state_dict.

    Returns (blob float32 1-D, n_out).
    """
    sd = strip_module_prefix(sd) if any(k.startswith("module.") for k in sd) or "state_dict" in sd else sd
    check_state_dict(sd, kind)
    parts = []
    for slot, lin, bn in _ENCODER:
        Wt, b = _fold(sd, lin, bn)
        if slot == "S3_F3":
            b = b + np.eye(3).reshape(-1)     # pointnet2.py:183-184  x + iden
        if slot == "SK_F3":
            b = b + np.eye(64).reshape(-1)    # pointnet2.py:221-222
        parts += [_pad64(Wt), _pad64(b)]
    if kind == "cls":
        for lin, bn in [("fc1", "bn1"), ("fc2", "bn2"), ("fc3", None)]:   # pointnet2.py:295-298
            Wt, b = _fold(sd, lin, bn)
            parts += [_pad64(Wt), _pad64(b)]
        n_out = Wt.shape[1]
        parts += [np.zeros(0, np.float32)] * 4   # HEAD3, HEAD4 are empty for cls
    elif kind == "seg":
        Wt, b = _fold(sd, "conv1", "bn1")        # (1088, 512): rows 0..1023 global, 1024..1087 point (pointnet2.py:270-271)
        parts += [_pad64(Wt[:1024]), _pad64(b)]  # HEAD0: global half carries the bias
        parts += [_pad64(Wt[1024:]), _pad64(np.zeros(512))]  # HEAD1: point half
        for lin, bn in [("conv2", "bn2"), ("conv3", "bn3"), ("conv4", None)]:
            Wt, b = _fold(sd, lin, bn)
            parts += [_pad64(Wt), _pad64(b)]
        n_out = Wt.shape[1]
    else:
        raise ValueError(kind)
    return np.concatenate(parts).astype(np.float32), int(n_out)
