"""Prediction-point sharding across the GPUs of one box, one process per GPU (SURVEY.md §8e).

Every prediction point is independent given the factorisation (ok.py:679-681 is column-wise
independent; the moving window is independent per point, ok.py:732-756), so the flattened work list is
cut into contiguous blocks, one per rank. Rank 0 assembles and factors; ONE broadcast (NCCL over
NVLink) ships the factor blob — packed inverse Cholesky factor, dual rows, drift constants, adjusted
data coordinates; no other collective is on the data path (a one-integer status precedes it so that a
failed factorisation raises on every rank instead of hanging the collective). The moving window
broadcasts nothing: every rank builds its own cell grid from the coordinates. torch is used only as the
owner of the process group and as a zero-copy view of the blob's device memory.

The single-process variant (one host thread, ``execute(..., n_gpus=G)``) lives behind the C ABI
(``kb200_group_*``, csrc/api.cu) and needs no process group.
"""
import numpy as np

from . import _cabi


def shard_range(count, rank, world):
    """Contiguous block [first, first+n) of `count` items for `rank` of `world` (sizes differ by <= 1)."""
    count, rank, world = int(count), int(rank), int(world)
    base, rem = divmod(count, world)
    first = rank * base + min(rank, rem)
    return first, base + (1 if rank < rem else 0)


class _DevicePtr:
    """Minimal __cuda_array_interface__ carrier so torch can view library-owned device memory."""

    def __init__(self, ptr, nbytes):
        self.__cuda_array_interface__ = {
            "shape": (int(nbytes),), "typestr": "|u1", "data": (int(ptr), False), "version": 2,
        }


def blob_as_tensor(handle, device):
    import torch

    ptr, nbytes = handle.blob()
    if not ptr or not nbytes:
        raise RuntimeError("the handle has no factor blob (describe/set the problem first)")
    return torch.as_tensor(_DevicePtr(ptr, nbytes), device=device)


def _active(dist):
    return dist is not None and dist.is_initialized() and dist.get_world_size() > 1


def prepare_sharded(model, dist=None, src=0, dtype="float64", device=None):
    """Make `model` ready to execute on every rank: rank `src` factors, everyone else only describes
    the problem (allocating the blob) and receives the broadcast. Returns the model's C-ABI handle.
    A failure on `src` (singular matrix, out of memory, unsupported dtype) is re-raised on every rank."""
    if not _active(dist):
        return model._ensure_problem(dtype)
    import torch

    rank = dist.get_rank()
    dev = device if device is not None else torch.device("cuda", torch.cuda.current_device())
    status = torch.zeros(1, dtype=torch.int32, device=dev)
    err = None
    h = None
    if rank == src:
        try:
            h = model._ensure_problem(dtype)
        except Exception as e:  # noqa: BLE001  (reported to every rank below)
            err = e
            status += 1
    else:
        try:                              # record the problem and allocate the blob, no device work
            h = model._cuda_handle()
            model._kb_key = None
            model._set_up_problem(h, _cabi.dtype_code(dtype), describe_only=True)
        except Exception as e:  # noqa: BLE001
            err = e
    dist.broadcast(status, src=src)      # one integer: did the factorisation succeed?
    if int(status.item()) != 0:
        if err is not None:
            raise err
        raise RuntimeError("rank %d failed to factor the kriging system (see its traceback)" % src)
    if err is not None:
        raise err
    t = blob_as_tensor(h, dev)
    dist.broadcast(t, src=src)           # the single data collective of the path
    if torch.device(dev).type == "cuda":
        torch.cuda.current_stream().synchronize()
    if rank != src:
        h.blob_commit()
        model._kb_key = model._problem_key(_cabi.dtype_code(dtype), False)
    return h


def execute_sharded(model, style, axes, dist=None, mask=None, n_closest_points=None, dtype="float64",
                    drift_at=None, gather=False, device=None):
    """This rank's contiguous block of one execute() call, any style:

      style 'grid' | 'masked' | 'points', axes = [x, y(, z)] grid axes or point lists (original coordinates),
      mask = flattened bool mask for 'masked', n_closest_points = moving window, drift_at = the host drift
      callback of UniversalKriging(3D).execute.

    Returns (z, ss, first, count): host arrays of the block and its position in the work list ('masked': the
    list of unmasked cells). With gather=True every rank returns the complete flat (z, ss) in the reference's
    order instead (all_gather_object; for tests and small jobs — the data path itself needs no gather)."""
    model._cover_prediction_points(axes)
    if n_closest_points is not None:
        h = model._ensure_problem("float64", knn=True)       # coordinates only: every rank builds its own cell grid
    else:
        h = prepare_sharded(model, dist, dtype=dtype, device=device)
    plan = model._plan(style, [np.asarray(a, dtype=np.float64) for a in axes], mask, drift_at)
    if _active(dist):
        first, count = shard_range(plan["count"], dist.get_rank(), dist.get_world_size())
    else:
        first, count = 0, plan["count"]
    z, ss = model._run_block(h, plan, first, count, n_closest_points, drift_at)
    if not gather:
        return z, ss, first, count
    if _active(dist):
        parts = [None] * dist.get_world_size()
        dist.all_gather_object(parts, (first, z, ss))
        parts.sort(key=lambda p: p[0])
        z = np.concatenate([p[1] for p in parts])
        ss = np.concatenate([p[2] for p in parts])
    return model._scatter(plan, z, ss)

