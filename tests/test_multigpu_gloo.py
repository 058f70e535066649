"""world_size-2 gloo tests (CPU) of the N>1 host path (pykrige_b200.multigpu): rank 0 factors, a one-integer
status and ONE broadcast of the factor blob follow, the non-root ranks only describe the problem and commit the
received blob, every rank executes its contiguous block of the work list (grid / masked / points), the gathered
blocks equal the single-process result. The device executor is replaced by a CPU stub built on the oracle (the
C-ABI handle needs a GPU); everything else — prepare_sharded, describe/commit order, plan / block / scatter,
error propagation — is the product code."""
import os
import socket
import sys
import numpy as np
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


class StubHandle:
    """CPU stand-in for _cabi.Handle: the 'factor blob' is the dense inverse of the reference's kriging matrix
    (oracle), execution is inverse x RHS on this rank's block. Records the call order."""

    def __init__(self, device=-1):
        self.calls = []
        self.blob_t = None
        self.ready = False

    def set_coordinates(self, geo): self.calls.append("coords")
    def set_pseudo_inverse(self, on): self.calls.append("pinv")
    def set_device_drift(self, wells, ext): self.calls.append("devdrift")
    def set_stream(self, s): pass

    def _remember(self, dim, x, y, values, model_id, vparams):
        self.xyz = np.column_stack([x, y])
        self.values = np.asarray(values, float)
        self.stored = list(vparams)

    def describe_problem(self, dim, dtype, x, y, z, values, center, aniso, model, vparams, exact, eps, n_rl=0, drift_data=None):
        self.calls.append("describe")
        self._remember(dim, x, y, values, model, vparams)
        n = len(x)
        self.blob_t = torch.zeros((n + 1) * (n + 1), dtype=torch.float64)

    def set_problem(self, dim, dtype, x, y, z, values, center, aniso, model, vparams, exact, eps, n_rl=0, drift_data=None):
        import scipy.linalg
        from oracle import krige_oracle as ko
        self.calls.append("set_problem")
        self._remember(dim, x, y, values, model, vparams)
        if len(np.unique(self.xyz, axis=0)) < len(self.xyz):
            raise np.linalg.LinAlgError("singular matrix")
        a = ko.kriging_matrix(self.xyz, "exponential", self.stored)
        self.blob_t = torch.from_numpy(scipy.linalg.inv(a).ravel().copy())
        self.ready = True

    def blob_commit(self):
        self.calls.append("commit")
        self.ready = True

    def _krige(self, Q):
        from scipy.spatial.distance import cdist
        from oracle import krige_oracle as ko
        assert self.ready
        n = self.xyz.shape[0]
        a_inv = self.blob_t.numpy().reshape(n + 1, n + 1)
        bd = cdist(Q, self.xyz)
        b = np.ones((Q.shape[0], n + 1))
        b[:, :n] = -ko.variogram("exponential", self.stored, bd)
        b[:, :n][np.abs(bd) <= 1e-10] = 0.0
        x = a_inv @ b.T
        return x[:n].T @ self.values, -np.einsum("ij,ji->i", b, x)

    def execute_grid(self, gx, gy, gz=None, drift=None, first=0, count=None):
        from oracle import krige_oracle as ko
        G = ko.grid_points([np.asarray(gx), np.asarray(gy)])
        return self._krige(G[first:first + count])

    def execute_points(self, px, py, pz=None, drift=None):
        return self._krige(np.column_stack([px, py]))


def _worker(rank, world, port, outdir):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    import cases
    import pykrige_b200 as pk
    from pykrige_b200 import multigpu, _cabi

    _cabi.Handle = StubHandle                                   # the only stubbed piece: the device executor
    multigpu.blob_as_tensor = lambda h, device: h.blob_t
    cpu = torch.device("cpu")
    xyz, val = cases.synth_data(42, 120, 2)
    gx, gy = np.linspace(0, 1000, 17), np.linspace(0, 1000, 13)
    rng = np.random.default_rng(3)
    mask = rng.uniform(size=(gy.size, gx.size)) < 0.4
    px, py = rng.uniform(0, 1000, 101), rng.uniform(0, 1000, 101)
    out = {}
    for name, style, axes, kw in (("grid", "grid", [gx, gy], {}), ("masked", "masked", [gx, gy], {"mask": mask.flatten()}),
                                  ("points", "points", [px, py], {})):
        m = pk.OrdinaryKriging(xyz[:, 0], xyz[:, 1], val, variogram_model="exponential", variogram_parameters=[1.0, 300.0, 0.05])
        z, ss, first, count = multigpu.execute_sharded(m, style, axes, dist, device=cpu, **kw)
        zf, sf = multigpu.execute_sharded(m, style, axes, dist, device=cpu, gather=True, **kw)
        out[name + "_z"], out[name + "_ss"], out[name + "_first"], out[name + "_count"] = z, ss, first, count
        out[name + "_zf"], out[name + "_sf"] = zf, sf
        out[name + "_calls"] = np.array(",".join(m._kb_handle.calls))
    # a singular system on rank 0 raises on every rank instead of hanging the broadcast
    dup = np.vstack([xyz[:10], xyz[:10]])
    bad = pk.OrdinaryKriging(dup[:, 0], dup[:, 1], np.concatenate([val[:10], val[:10]]), variogram_model="exponential",
                             variogram_parameters=[1.0, 300.0, 0.05])
    try:
        multigpu.execute_sharded(bad, "grid", [gx, gy], dist, device=cpu)
        out["raised"] = np.array(0)
    except (np.linalg.LinAlgError, RuntimeError):
        out["raised"] = np.array(1)
    np.savez(os.path.join(outdir, "r%d.npz" % rank), **out)
    dist.barrier()
    dist.destroy_process_group()


def test_shard_range_covers_everything():
    sys.path.insert(0, ROOT)
    from pykrige_b200 import multigpu
    for count in (0, 1, 7, 100, 1000003):
        for world in (1, 2, 3, 8):
            blocks = [multigpu.shard_range(count, r, world) for r in range(world)]
            assert blocks[0][0] == 0 and sum(c for _, c in blocks) == count
            for (f0, c0), (f1, c1) in zip(blocks, blocks[1:]):
                assert f1 == f0 + c0 and 0 <= c0 - c1 <= 1


def test_two_rank_sharding_matches_single(tmp_path):
    world = 2
    port = _free_port()
    mp.spawn(_worker, args=(world, port, str(tmp_path)), nprocs=world, join=True)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import cases
    from oracle import krige_oracle as ko
    xyz, val = cases.synth_data(42, 120, 2)
    gx, gy = np.linspace(0, 1000, 17), np.linspace(0, 1000, 13)
    rng = np.random.default_rng(3)
    mask = rng.uniform(size=(gy.size, gx.size)) < 0.4
    px, py = rng.uniform(0, 1000, 101), rng.uniform(0, 1000, 101)
    stored = ko.stored_parameters("exponential", [1.0, 300.0, 0.05])
    G = ko.grid_points([gx, gy])
    parts = [np.load(os.path.join(str(tmp_path), "r%d.npz" % r)) for r in range(world)]
    work = {"grid": G, "masked": G[~mask.flatten()], "points": np.column_stack([px, py])}
    for name, Q in work.items():
        z1, s1 = ko.krige(xyz, val, "exponential", stored, Q)
        assert parts[0][name + "_first"] == 0
        assert parts[0][name + "_count"] + parts[1][name + "_count"] == Q.shape[0]
        assert parts[1][name + "_first"] == parts[0][name + "_count"]
        z = np.concatenate([p[name + "_z"] for p in parts])
        ss = np.concatenate([p[name + "_ss"] for p in parts])
        np.testing.assert_allclose(z, z1, rtol=1e-10)
        np.testing.assert_allclose(ss, s1, rtol=1e-9, atol=1e-12)
        # gather=True: every rank holds the complete result in the reference's flattened order
        for p in parts:
            zf, sf = p[name + "_zf"], p[name + "_sf"]
            if name == "masked":
                assert zf.size == G.shape[0] and np.all(zf[mask.flatten()] == 0.0)
                zf, sf = zf[~mask.flatten()], sf[~mask.flatten()]
            np.testing.assert_allclose(zf, z1, rtol=1e-10)
            np.testing.assert_allclose(sf, s1, rtol=1e-9, atol=1e-12)
    # call order: rank 0 factors, rank 1 only describes and commits the broadcast blob
    c0, c1 = str(parts[0]["grid_calls"]), str(parts[1]["grid_calls"])
    assert "set_problem" in c0 and "describe" not in c0 and "commit" not in c0
    assert "describe" in c1 and "commit" in c1 and "set_problem" not in c1
    assert c1.index("devdrift") < c1.index("describe") < c1.index("commit")
    assert int(parts[0]["raised"]) == 1 and int(parts[1]["raised"]) == 1


# ---- second worker: the full-surface C-ABI emulator (tests/abi_emulator.py) instead of the minimal stub, so that the
#      sharded path is exercised for universal kriging (device-evaluated and host-supplied drift columns: the drift_at
#      callback receives the block's position in the caller's arrays), 3-D, the moving window and a custom variogram ----
def _emulated_jobs():
    import cases
    rng = np.random.default_rng(17)
    xyz, val = cases.synth_data(61, 90, 2)
    x3, v3 = cases.synth_data(62, 70, 3)
    gx, gy, gz = np.linspace(0, 1000, 11), np.linspace(0, 1000, 9), np.linspace(0, 250, 4)
    mask = rng.uniform(size=(gy.size, gx.size)) < 0.35
    mask3 = rng.uniform(size=(gz.size, gy.size, gx.size)) < 0.35
    px, py, pz = rng.uniform(0, 1000, 53), rng.uniform(0, 1000, 53), rng.uniform(0, 250, 53)
    dem = rng.uniform(0, 5, (8, 7))
    demx, demy = np.linspace(-10, 1010, 7), np.linspace(-10, 1010, 8)
    wells = np.array([[100.0, 200.0, 1.0], [700.0, 650.0, -2.0]])
    vp = dict(variogram_model="exponential", variogram_parameters=[1.0, 300.0, 0.05])
    uk_kw = dict(vp, drift_terms=["regional_linear", "point_log", "external_Z", "specified", "functional"],
                 point_drift=wells, external_drift=dem, external_drift_x=demx, external_drift_y=demy,
                 specified_drift=[1.0e-5 * xyz[:, 0] * xyz[:, 1]], functional_drift=[lambda x, y: np.sin(x / 300.0) * y / 1000.0],
                 anisotropy_scaling=1.4, anisotropy_angle=25.0)
    spec_grid = 1.0e-5 * gx[None, :] * gy[:, None]
    spec_pts = 1.0e-5 * px * py
    jobs = [
        ("uk_grid", "UniversalKriging", (xyz[:, 0], xyz[:, 1], val), uk_kw, ("grid", gx, gy), dict(specified_drift_arrays=[spec_grid])),
        # execute(values=...) first: its value fields must not stay on the handle of the rank that only describes
        ("uk_grid_after_fields", "UniversalKriging", (xyz[:, 0], xyz[:, 1], val), uk_kw, ("grid", gx, gy),
         dict(specified_drift_arrays=[spec_grid])),
        ("uk_masked", "UniversalKriging", (xyz[:, 0], xyz[:, 1], val), uk_kw, ("masked", gx, gy), dict(mask=mask, specified_drift_arrays=[spec_grid])),
        ("uk_points", "UniversalKriging", (xyz[:, 0], xyz[:, 1], val), uk_kw, ("points", px, py), dict(specified_drift_arrays=[spec_pts])),
        ("ok3d_masked", "OrdinaryKriging3D", (x3[:, 0], x3[:, 1], x3[:, 2], v3), vp, ("masked", gx, gy, gz), dict(mask=mask3)),
        ("uk3d_points", "UniversalKriging3D", (x3[:, 0], x3[:, 1], x3[:, 2], v3),
         dict(vp, drift_terms=["regional_linear", "functional"], functional_drift=[lambda x, y, z: x * z / 1.0e5]), ("points", px, py, pz), {}),
        ("ok_knn_grid", "OrdinaryKriging", (xyz[:, 0], xyz[:, 1], val), vp, ("grid", gx, gy), dict(n_closest_points=6)),
        ("ok_custom_points", "OrdinaryKriging", (xyz[:, 0], xyz[:, 1], val),
         dict(variogram_model="custom", variogram_parameters=[0.05, 0.1], variogram_function=lambda m, d: m[0] * np.sqrt(d) + m[1]),
         ("points", px, py), {}),
    ]
    return jobs


def _sharded_execute(model, multigpu, dist, args, kw, device):
    """What a caller of execute() does under torchrun: the class validates and plans, execute_sharded runs the block.
    Uses the public execute() with `_run_cuda` re-routed to the sharded executor (gather=True)."""
    def run_cuda(style, axes, mask, n_closest_points=None, drift_at=None, dtype="float64", n_gpus=None, fields=None):
        assert fields is None
        return multigpu.execute_sharded(model, style, axes, dist, mask=mask, n_closest_points=n_closest_points,
                                        dtype=dtype, drift_at=drift_at, gather=True, device=device)
    model._run_cuda = run_cuda
    return model.execute(*args, backend="cuda", **kw)


def _worker_emulated(rank, world, port, outdir):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    import pykrige_b200 as pk
    from pykrige_b200 import multigpu, _cabi
    from fields_emulator import FieldsEmulatedHandle

    def no_device():
        raise _cabi.KrigeB200Error("emulated box")

    _cabi.Handle = FieldsEmulatedHandle
    _cabi.aux_handle = no_device
    multigpu.blob_as_tensor = lambda h, device: h.blob_t
    cpu = torch.device("cpu")
    out = {}
    for name, cls, cargs, ckw, eargs, ekw in _emulated_jobs():
        m = getattr(pk, cls)(*cargs, **ckw)
        if name.endswith("_after_fields"):
            v = cargs[-1]
            m.execute(*eargs, backend="cuda", values=np.column_stack([v, v[::-1]]), **ekw)
            del m._kb_handle.calls[:]
        z, ss = _sharded_execute(m, multigpu, dist, eargs, ekw, cpu)
        out[name + "_z"], out[name + "_ss"] = np.ma.getdata(z), np.ma.getdata(ss)
        out[name + "_calls"] = np.array(",".join(m._kb_handle.calls))
    np.savez(os.path.join(outdir, "e%d.npz" % rank), **out)
    dist.barrier()
    dist.destroy_process_group()


def test_two_rank_sharding_of_every_problem_kind(tmp_path, monkeypatch):
    """2 gloo ranks vs one process, both through the C-ABI emulator: universal kriging with all five drift kinds
    (grid / masked / points — the host drift callback must be evaluated at the block's own positions; also after an
    execute(values=...) on the same objects), 3-D masked,
    UK3D points, the moving window (no broadcast) and a tabulated custom variogram (every rank tabulates itself)."""
    world = 2
    port = _free_port()
    mp.spawn(_worker_emulated, args=(world, port, str(tmp_path)), nprocs=world, join=True)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import pykrige_b200 as pk
    from pykrige_b200 import _cabi
    from fields_emulator import FieldsEmulatedHandle

    def no_device():
        raise _cabi.KrigeB200Error("emulated box")

    monkeypatch.setattr(_cabi, "Handle", FieldsEmulatedHandle)
    monkeypatch.setattr(_cabi, "aux_handle", no_device)
    parts = [np.load(os.path.join(str(tmp_path), "e%d.npz" % r)) for r in range(world)]
    for name, cls, cargs, ckw, eargs, ekw in _emulated_jobs():
        m = getattr(pk, cls)(*cargs, **ckw)
        z1, s1 = m.execute(*eargs, backend="cuda", **ekw)
        z1, s1 = np.ma.getdata(z1), np.ma.getdata(s1)
        for p in parts:                                      # gather=True: every rank holds the complete result
            assert p[name + "_z"].shape == z1.shape
            np.testing.assert_allclose(p[name + "_z"], z1, rtol=1e-9, atol=1e-9 * np.abs(z1).max(), err_msg=name)
            np.testing.assert_allclose(p[name + "_ss"], s1, rtol=1e-8, atol=1e-9 * np.abs(s1).max(), err_msg=name)
        c0, c1 = str(parts[0][name + "_calls"]), str(parts[1][name + "_calls"])
        if "knn" in name:                                    # the moving window broadcasts nothing
            assert "set_problem_knn" in c0 and "set_problem_knn" in c1 and "describe_problem" not in c1
        else:                                                # rank 0 factors, rank 1 describes + commits the broadcast
            assert "set_problem" in c0.split(",") and "describe_problem" not in c0
            assert "describe_problem" in c1 and "blob_commit" in c1 and "set_problem" not in c1.split(",")
        if name.endswith("_after_fields"):                   # the fields of the earlier run are dropped first
            assert c1.split(",")[0] == "set_values"
