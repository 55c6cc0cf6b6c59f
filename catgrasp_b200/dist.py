"""Multi-GPU plumbing: candidates shard across ranks, one all-gather of the result records.

The path partitions by candidate (SURVEY.md 8e): each rank scores a contiguous block
[lo, hi) of the B candidates against replicated cloud / SDF / weights (no data-path collective),
then a single ``all_gather`` of fixed-width 48-byte records (10 fp32 probabilities, status, offset,
pad) rebuilds the full, candidate-ordered result on every rank.  NCCL over NVLink on GPUs; the same
code runs over gloo on CPU tensors for the host-logic tests.
"""
import torch
import torch.distributed as dist

RECORD_FLOATS = 12   # 10 probs + [status, offset] packed as two floats = 48 bytes


def shard_range(n, rank, world):
    """Contiguous block of ceil(n/world) items per rank (keeps RNG-ordered ids aligned with candidate order)."""
    per = (n + world - 1) // world
    lo = min(n, rank * per)
    hi = min(n, lo + per)
    return lo, hi


def pack_records(probs, status, offset):
    """(b,10) f32, (b,) u8, (b,) i8 -> (b,12) f32 records."""
    b = probs.shape[0]
    rec = torch.zeros((b, RECORD_FLOATS), dtype=torch.float32, device=probs.device)
    rec[:, : probs.shape[1]] = probs
    rec[:, 10] = status.to(torch.float32)
    rec[:, 11] = offset.to(torch.float32)
    return rec


def unpack_records(rec, n_out=10):
    return rec[:, :n_out].contiguous(), rec[:, 10].to(torch.uint8), rec[:, 11].to(torch.int8)


def all_gather_records(local_rec, n_total, group=None):
    """Gather every rank's (b_r, 12) block into the full (n_total, 12) tensor, in candidate order.

    Blocks are padded to the common ceil(n/world) length so that one ``all_gather_into_tensor``
    (ncclAllGather) moves everything."""
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
        return local_rec[:n_total]
    world = dist.get_world_size(group)
    per = (n_total + world - 1) // world
    pad = torch.zeros((per, RECORD_FLOATS), dtype=local_rec.dtype, device=local_rec.device)
    pad[: local_rec.shape[0]] = local_rec
    out = torch.empty((world * per, RECORD_FLOATS), dtype=local_rec.dtype, device=local_rec.device)
    dist.all_gather_into_tensor(out, pad, group=group)
    return out[:n_total]


def sharded_predict_batch(predicter, data, grasp_poses, subsample=None, group=None):
    """``GraspPredicter.predict_batch(data, grasp_poses)`` (predicter.py:67-94) with the candidate list sharded over the
    ranks of ``group``: every rank calls this with the SAME arguments, scores its contiguous block
    (``predicter.score(..., shard=shard_range(B, rank, world))``) against the replicated cloud and weights, and one
    all-gather of the (B, 12) records rebuilds the full, candidate-ordered result on every rank.  Same return value as predict_batch; with
    ``subsample="host"`` every rank consumes the global numpy generator exactly like the single-process call."""
    from .predicter import result_list
    B = len(grasp_poses)
    if B == 0:
        return []
    world = dist.get_world_size(group) if (dist.is_available() and dist.is_initialized()) else 1
    rank = dist.get_rank(group) if world > 1 else 0
    d_probs = predicter.score(data, grasp_poses, subsample=subsample, shard=shard_range(B, rank, world))
    zero = torch.zeros((d_probs.shape[0],), device=d_probs.device)    # scoring has no status or offset: both columns 0
    full = all_gather_records(pack_records(d_probs, zero, zero), B, group=group)
    return result_list(unpack_records(full, d_probs.shape[1])[0].cpu().numpy())
