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


# ---- PointGroup (PointGroup/model/pointgroup/pointgroup.py) ----
# spconv 1.x stores a convolution's weight as (k, k, k, Cin, Cout).  Every BatchNorm1d sits in front of a convolution
# (BN, ReLU, conv), so it cannot be folded into the conv's weights; it is kept as a per-channel (scale, shift), which
# the conv kernel applies to present rows only.  The offset head's BN follows its first Linear and is folded into it.

PG_INPUT_C = 6          # normals + coordinates (input_channel 3, use_coords)
PG_LEVELS = 7           # UBlock([m, 2m, ..., 7m])


def _pg_bn(keys, p, C):
    for s in (".weight", ".bias", ".running_mean", ".running_var"):
        keys[p + s] = (C,)


def _pg_conv(keys, p, k, cin, cout):
    keys[p + ".weight"] = (k, k, k, cin, cout)
    keys[p + ".bias"] = (cout,)


def _pg_resblock(keys, p, cin, cout):
    if cin != cout:
        _pg_conv(keys, p + "i_branch.0", 1, cin, cout)
    _pg_bn(keys, p + "conv_branch.0", cin)
    _pg_conv(keys, p + "conv_branch.2", 3, cin, cout)
    _pg_bn(keys, p + "conv_branch.3", cout)
    _pg_conv(keys, p + "conv_branch.5", 3, cout, cout)


def _pg_ublock(keys, p, planes, reps):
    for i in range(reps):
        _pg_resblock(keys, f"{p}blocks.block{i}.", planes[0], planes[0])
    if len(planes) > 1:
        _pg_bn(keys, p + "conv.0", planes[0])
        _pg_conv(keys, p + "conv.2", 2, planes[0], planes[1])
        _pg_ublock(keys, p + "u.", planes[1:], reps)
        _pg_bn(keys, p + "deconv.0", planes[1])
        _pg_conv(keys, p + "deconv.2", 2, planes[1], planes[0])
        for i in range(reps):
            _pg_resblock(keys, f"{p}blocks_tail.block{i}.", planes[0] * (2 - i), planes[0])


def pointgroup_keys(m, block_reps):
    """The parameter and buffer names of PointGroup(m, block_reps) with residual blocks and use_coords, and their
    shapes, in module order (num_batches_tracked left out).  The score branch's keys are included: the reference
    loads strictly, although inference never runs that branch."""
    keys = OrderedDict()
    _pg_conv(keys, "input_conv.0", 3, PG_INPUT_C, m)
    _pg_ublock(keys, "unet.", [m * (i + 1) for i in range(PG_LEVELS)], block_reps)
    _pg_bn(keys, "output_layer.0", m)
    keys["offset.0.weight"], keys["offset.0.bias"] = (m, m), (m,)
    _pg_bn(keys, "offset.1", m)
    keys["offset.3.weight"], keys["offset.3.bias"] = (3, m), (3,)
    _pg_ublock(keys, "score_unet.", [m, 2 * m], 2)
    _pg_bn(keys, "score_outputlayer.0", m)
    keys["score_linear.weight"], keys["score_linear.bias"] = (1, m), (1,)
    return keys


def check_pointgroup_state_dict(sd, m, block_reps):
    """Strict check of a PointGroup state_dict: raises RuntimeError naming the missing or unexpected keys, or
    ValueError naming the first key whose shape is wrong."""
    want = pointgroup_keys(m, block_reps)
    have = [k for k in sd.keys() if not k.endswith("num_batches_tracked")]
    missing, extra = [k for k in want if k not in sd], sorted(set(have) - set(want))
    if missing or extra:
        raise RuntimeError(f"checkpoint does not match PointGroup(m={m}, block_reps={block_reps}): "
                           f"missing={missing[:8]} unexpected={extra[:8]}")
    for k, shape in want.items():
        got = tuple(sd[k].shape)
        if got != shape:
            raise ValueError(f"checkpoint key {k} has shape {got}, PointGroup(m={m}, block_reps={block_reps}) "
                             f"expects {shape}")


def _bn_affine(sd, p):
    """Eval-mode BatchNorm1d as y = x * scale + shift, computed in float64 and narrowed to float32."""
    g, beta = _np64(sd[p + ".weight"]), _np64(sd[p + ".bias"])
    mu, var = _np64(sd[p + ".running_mean"]), _np64(sd[p + ".running_var"])
    s = g / np.sqrt(var + BN_EPS)
    return np.float32(s), np.float32(beta - mu * s)


def _f32(sd, k, K=None):
    a = _np64(sd[k]).astype(np.float32)
    return np.ascontiguousarray(a if K is None else a.reshape(K, a.shape[-2], a.shape[-1]))


def _pack_resblock(sd, p, cin, cout):
    blk = {"bn1": _bn_affine(sd, p + "conv_branch.0"),
           "W1": _f32(sd, p + "conv_branch.2.weight", 27), "b1": _f32(sd, p + "conv_branch.2.bias"),
           "bn2": _bn_affine(sd, p + "conv_branch.3"),
           "W2": _f32(sd, p + "conv_branch.5.weight", 27), "b2": _f32(sd, p + "conv_branch.5.bias"),
           "Wi": None, "bi": None}
    if cin != cout:
        blk["Wi"], blk["bi"] = _f32(sd, p + "i_branch.0.weight", 1), _f32(sd, p + "i_branch.0.bias")
    return blk


def pack_pointgroup(sd, m, block_reps):
    """The float32 arrays the device forward runs on, from a PointGroup state_dict (``module.`` prefixes and a
    'state_dict' wrapper are stripped; the key set and shapes are checked strictly).  Returns a dict:
      input: (W (27,6,m), b); levels: one dict per level l = 0..6 with C = (l+1) m and
        blocks / tail: lists of residual blocks {bn1: (scale, shift), W1 (27,Cin,C), b1, bn2, W2 (27,C,C), b2,
        Wi (1,Cin,C) or None, bi}, and for l < 6 down: (bn, W (8,C,C+m), b), up: (bn, W (8,C+m,C), b);
      head: {bn: output_layer's (scale, shift), W1 (m,m) [in][out] and b1 with offset.1 folded in, W2 (m,3), b2}."""
    if any(k.startswith("module.") for k in sd) or "state_dict" in sd:
        sd = strip_module_prefix(sd)
    check_pointgroup_state_dict(sd, m, block_reps)
    out = {"input": (_f32(sd, "input_conv.0.weight", 27), _f32(sd, "input_conv.0.bias")), "levels": []}
    p = "unet."
    for lv in range(PG_LEVELS):
        C = m * (lv + 1)
        L = {"blocks": [_pack_resblock(sd, f"{p}blocks.block{i}.", C, C) for i in range(block_reps)]}
        if lv < PG_LEVELS - 1:
            L["down"] = (_bn_affine(sd, p + "conv.0"), _f32(sd, p + "conv.2.weight", 8), _f32(sd, p + "conv.2.bias"))
            L["up"] = (_bn_affine(sd, p + "deconv.0"), _f32(sd, p + "deconv.2.weight", 8),
                       _f32(sd, p + "deconv.2.bias"))
            L["tail"] = [_pack_resblock(sd, f"{p}blocks_tail.block{i}.", C * (2 - i), C) for i in range(block_reps)]
        out["levels"].append(L)
        p += "u."
    W1, b1 = _fold(sd, "offset.0", "offset.1")
    W2, b2 = _fold(sd, "offset.3", None)
    out["head"] = {"bn": _bn_affine(sd, "output_layer.0"), "W1": np.float32(W1), "b1": np.float32(b1),
                   "W2": np.float32(W2), "b2": np.float32(b2)}
    return out
