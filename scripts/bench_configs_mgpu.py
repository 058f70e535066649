"""BASELINE.json configs 3, 4, 5 at their named GPU counts (torchrun, one rank per GPU):
    cfg3  OK3D  N=8000,  200x200x50 grid, gaussian,  fp64,               all ranks (named: 8 GPUs)
    cfg4  UK2D  N=10000, 2000x2000 grid,  exponential, fp32 (3xTF32),    first 4 ranks (named: 4 GPUs)
    cfg5  OK2D  N=100000, 4000x4000 grid, k=64 moving window, fp64,      all ranks (named: 8 GPUs)
Whole grids, points sharded contiguously, rank 0 factors + ONE broadcast (global path); the moving window
needs no collective (every rank builds its own cell grid). Time = max over ranks (barrier-bracketed wall
clock of the host-buffer API, so H2D/D2H are inside). Rank 0 prints one JSON line per config."""
import json
import os
import sys
import time
import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import cases  # noqa: E402
import pykrige_b200 as pk  # noqa: E402
from pykrige_b200 import multigpu  # noqa: E402

rank = int(os.environ.get("RANK", "0"))
world = int(os.environ.get("WORLD_SIZE", "1"))
local = int(os.environ.get("LOCAL_RANK", "0"))
saved = os.dup(1)
os.dup2(2, 1)
torch.cuda.set_device(local)
dist.init_process_group("nccl", device_id=torch.device("cuda", local))
sub4 = dist.new_group(list(range(min(4, world))))


def emit(obj):
    if rank == 0:
        sys.stdout.flush()
        os.dup2(saved, 1)
        print(json.dumps(obj), flush=True)
        os.dup2(2, 1)


def timed(fn, group, nranks):
    dist.barrier(group=group)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    dt = torch.tensor([time.perf_counter() - t0], dtype=torch.float64, device="cuda")
    dist.all_reduce(dt, op=dist.ReduceOp.MAX, group=group)
    return float(dt.item()), out


class _Sub:
    """torch.distributed facade restricted to a sub-group (for multigpu.prepare_sharded)."""
    def __init__(self, group, n):
        self.group, self.n = group, n
    def is_initialized(self): return True
    def get_world_size(self): return self.n
    def get_rank(self): return dist.get_rank(self.group)
    def broadcast(self, t, src=0): return dist.broadcast(t, src=src, group=self.group)


def run_global(name, model, axes, dtype, group, nranks, flop_pt):
    d = _Sub(group, nranks)
    npt = int(np.prod([a.size for a in axes]))
    def step():
        model._kb_key = None
        return multigpu.execute_sharded(model, "grid", axes, d, dtype=dtype)
    step()                                   # warm-up (allocations, first factorisation)
    dt, (z, ss, first, count) = timed(step, group, nranks)
    emit({"config": name, "n_gpus": nranks, "dtype": dtype, "grid_points": npt, "seconds_max_over_ranks": dt,
          "points_per_s_e2e": npt / dt, "algorithmic_tflops": npt * flop_pt / dt / 1e12,
          "z_mean_rank0_slice": float(np.mean(z)), "ss_mean_rank0_slice": float(np.mean(ss))})


if True:
    xyz, val = cases.synth_data(1003, 8000, 3)
    axes = [np.linspace(0, 1000, 200), np.linspace(0, 1000, 200), np.linspace(0, 250, 50)]
    m = pk.OrdinaryKriging3D(xyz[:, 0], xyz[:, 1], xyz[:, 2], val, variogram_model="gaussian", variogram_parameters=[1.0, 300.0, 0.05])
    run_global("cfg3", m, axes, "float64", dist.group.WORLD, world, 2.0 * 8001**2)
    del m

if rank < min(4, world):
    xyz, val = cases.synth_data(1004, 10000, 2)
    axes = [np.linspace(0, 1000, 2000), np.linspace(0, 1000, 2000)]
    m = pk.UniversalKriging(xyz[:, 0], xyz[:, 1], val, variogram_model="exponential", variogram_parameters=[1.0, 300.0, 0.05],
                            drift_terms=["regional_linear"])
    run_global("cfg4", m, axes, "float32", sub4, min(4, world), 2.0 * 10003**2)
    del m
dist.barrier()

if True:
    xyz, val = cases.synth_data(1005, 100000, 2)
    axes = [np.linspace(0, 1000, 4000), np.linspace(0, 1000, 4000)]
    m = pk.OrdinaryKriging(xyz[:, 0], xyz[:, 1], val, variogram_model="exponential", variogram_parameters=[1.0, 50.0, 0.05])
    npt = 4000 * 4000
    first, count = multigpu.shard_range(npt, rank, world)
    def step():
        m._kb_key = None
        h = m._ensure_problem("float64", knn=True)
        return h.execute_knn_grid(64, axes[0], axes[1], None, first, count)
    step()
    dt, (z, ss) = timed(step, dist.group.WORLD, world)
    emit({"config": "cfg5", "n_gpus": world, "dtype": "float64", "grid_points": npt, "k": 64, "seconds_max_over_ranks": dt,
          "points_per_s_e2e": npt / dt, "z_mean_rank0_slice": float(np.mean(z)), "ss_mean_rank0_slice": float(np.mean(ss))})

dist.barrier()
dist.destroy_process_group()
