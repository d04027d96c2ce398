"""-m gpu: ShardedLayer.exchange() keeps read-only replicas of the other ranks' blocks GPU to GPU, and every
consumer of the map on any rank -- the incremental and full mesh, the ESDF, ICP -- then gives the single-GPU
result.

Most cases run the W engines of a W-way sharded map on ONE GPU, each rank's exchange on a thread of its own,
joined by the in-process all-gather (sharded.LocalAllGather); the last case runs two processes over NCCL
when two GPUs are visible."""
import os
import socket
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import voxblox_b200 as vb
from voxblox_b200 import api, scenes, sharded
from tests import esdf_fixed_point as fp
from tests.test_icp_gpu import PERTURBATIONS, _perturbed

pytestmark = pytest.mark.gpu

CFG = dict(default_truncation_distance=0.4, integrator_threads=1)
OPTS = dict(max_blocks=4096, max_updates_per_pass=1 << 22)
ALL = api.UPDATED_MAP | api.UPDATED_MESH | api.UPDATED_ESDF
# Share of observed ESDF voxels whose distance on a rank differs from the single-GPU layer by more than 1e-4
# (mixed-sign voxels, whose outcome is a warp race: DESIGN.md section 6); measured bound, DESIGN.md section 8
MAX_DISTANCE_SHARE = 0.04  # (largest measured: 0.0315, W = 8, min_diff_m = 0)


def _scans(n=3):
    return scenes.c3_room_sequence(n_scans=n, width=160, height=120)


class Rank:
    def __init__(self, rank, world, gather, voxel=0.1, vps=16, trunc=0.4, opts=OPTS, esdf=None, mesh=False):
        self.rank = rank
        self.layer = vb.Layer(voxel, vps, engine_options=sharded.shard_options(rank, world, **opts))
        self.integ = vb.TsdfIntegratorFactory.create(
            2, vb.TsdfIntegratorConfig(default_truncation_distance=trunc, integrator_threads=1), self.layer)
        self.sl = sharded.ShardedLayer(self.layer, all_gather=gather.rank(rank))
        if esdf is not None:
            self.esdf = vb.Layer(voxel, vps, voxel_type="esdf")
            self.eint = vb.EsdfIntegrator(vb.EsdfIntegratorConfig(**esdf), self.layer, self.esdf)
        if mesh:
            self.mesh = vb.MeshLayer(self.layer.block_size())
            self.mint = vb.MeshIntegrator(vb.MeshIntegratorConfig(), self.layer, self.mesh)

    def owned(self, idx):
        return sharded.block_owner(idx, self.sl.world) == self.rank


def _ranks(world, **kw):
    gather = sharded.LocalAllGather(world)
    return [Rank(r, world, gather, **kw) for r in range(world)]


def _exchange(ranks):
    """Every rank's exchange() on its own thread: the blocks each received (an exception is re-raised)."""
    with ThreadPoolExecutor(len(ranks)) as ex:
        futs = [ex.submit(r.sl.exchange) for r in ranks]
        return [f.result() for f in futs]


def _single(voxel=0.1, vps=16, trunc=0.4, opts=OPTS, esdf=None, mesh=False):
    class S:
        pass

    s = S()
    s.layer = vb.Layer(voxel, vps, engine_options=vb.EngineOptions(**opts))
    s.integ = vb.TsdfIntegratorFactory.create(
        2, vb.TsdfIntegratorConfig(default_truncation_distance=trunc, integrator_threads=1), s.layer)
    if esdf is not None:
        s.esdf = vb.Layer(voxel, vps, voxel_type="esdf")
        s.eint = vb.EsdfIntegrator(vb.EsdfIntegratorConfig(**esdf), s.layer, s.esdf)
    if mesh:
        s.mesh = vb.MeshLayer(s.layer.block_size())
        s.mint = vb.MeshIntegrator(vb.MeshIntegratorConfig(), s.layer, s.mesh)
    return s


def _layer_state(layer):
    idx = layer.getAllAllocatedBlocks()
    vox, upd = layer.getBlocks(idx)
    return idx, vox, upd


def _assert_same_map(layer, ref_idx, ref_vox, what):
    idx, vox, _ = _layer_state(layer)
    assert idx.tolist() == ref_idx.tolist(), f"{what}: block set differs"
    assert vox.tobytes() == ref_vox.tobytes(), f"{what}: voxels differ"


# ---------------------------------------------------------------- 1. replicas
def _check_replicas(ranks, single, got):
    ref_idx, ref_vox, _ = _layer_state(single.layer)
    for rk in ranks:
        _assert_same_map(rk.layer, ref_idx, ref_vox, f"rank {rk.rank}")
        idx, _, upd = _layer_state(rk.layer)
        theirs = ~rk.owned(idx)
        # replicas carry what a scan gives a block; nothing of the mirror mark is left on the owned blocks
        assert (upd[theirs & (upd != 0)] == ALL).all()
        assert rk.layer.gatherUpdatedDevice(api.UPDATED_MIRROR, owned_only=True) == 0
    return ref_idx


@pytest.mark.parametrize("world", [2, 3, 8])
def test_replicas_equal_the_single_gpu_map(world):
    single = _single()
    ranks = _ranks(world)
    for k, s in enumerate(_scans(4)):
        single.integ.integratePointCloud((s[2], s[3]), s[0], s[1])
        before = {}
        for rk in ranks:
            rk.integ.integratePointCloud((s[2], s[3]), s[0], s[1])
            idx, vox, upd = _layer_state(rk.layer)
            before[rk.rank] = (idx, vox, upd)
            if k:
                # the scan left every replica's payload and (cleared) flags as the last exchange left them
                prev_idx, prev_vox = rk.after
                theirs = ~rk.owned(idx)
                assert idx[theirs].tolist() == prev_idx.tolist()
                assert vox[theirs].tobytes() == prev_vox.tobytes()
                assert (upd[theirs] == 0).all(), "a scan set updated bits on a block this rank does not own"
        got = _exchange(ranks)
        print("world", world, "scan", k, "blocks received per rank", got)
        assert sum(got) > 0
        _check_replicas(ranks, single, got)
        for rk in ranks:
            idx, _, upd = _layer_state(rk.layer)
            mine = rk.owned(idx)
            b_idx, _, b_upd = before[rk.rank]
            # the owner's reported bits are untouched by the exchange
            b_mine = rk.owned(b_idx)
            assert idx[mine].tolist() == b_idx[b_mine].tolist() and (upd[mine] == b_upd[b_mine]).all()
            # the replicas received now carry all three bits, the others are as the last exchange left them
            assert int((upd[~mine] == ALL).sum()) == got[rk.rank]
        assert _exchange(ranks) == [0] * world, "a second exchange without a scan moved blocks"
        for rk in ranks:
            rk.layer.clearUpdated(0), rk.layer.clearUpdated(1), rk.layer.clearUpdated(2)
            idx, vox, _ = _layer_state(rk.layer)
            theirs = ~rk.owned(idx)
            rk.after = (idx[theirs], vox[theirs])


def test_replicas_with_asynchronous_submission():
    world = 3
    single = _single()
    ranks = _ranks(world)
    keep = []
    scans = list(_scans(6))
    for k in range(0, len(scans), 2):
        for s in scans[k:k + 2]:
            single.integ.integratePointCloud((s[2], s[3]), s[0], s[1])
            p, c = np.ascontiguousarray(s[0]), np.ascontiguousarray(s[1])
            keep.append((p, c))
            for rk in ranks:
                rk.integ.integratePointCloudAsync((s[2], s[3]), p, c)
        got = _exchange(ranks)  # (every engine call drains the queued scans first)
        _check_replicas(ranks, single, got)
        assert _exchange(ranks) == [0] * world


def test_replicas_with_more_than_65535_blocks_on_one_rank():
    """C5 (two lidar scans) at vps 2: ~228 k blocks, so each of the two ranks gathers and receives more blocks
    than a grid's y dimension can number."""
    world, vps = 2, 2
    opts = dict(max_blocks=1 << 19)
    single = _single(voxel=0.05, vps=vps, trunc=0.2, opts=opts)
    ranks = _ranks(world, voxel=0.05, vps=vps, trunc=0.2, opts=opts)
    for i in range(2):
        s = scenes.c5_lidar_scan(i)
        single.integ.integratePointCloud((s[2], s[3]), s[0], s[1])
        for rk in ranks:
            rk.integ.integratePointCloud((s[2], s[3]), s[0], s[1])
    got = _exchange(ranks)
    print("blocks received per rank", got)
    assert min(got) > 65535
    _check_replicas(ranks, single, got)
    assert _exchange(ranks) == [0] * world


# ---------------------------------------------------------------- 2. mesh
def _assert_same_meshes(a: vb.MeshLayer, b: vb.MeshLayer, what):
    ka, kb = a.getAllAllocatedMeshes().tolist(), b.getAllAllocatedMeshes().tolist()
    assert ka == kb, f"{what}: mesh block set differs"
    for k in ka:
        ma, mb = a.getMeshPtrByIndex(k), b.getMeshPtrByIndex(k)
        for f in ("vertices", "normals", "colors"):
            assert getattr(ma, f).tobytes() == getattr(mb, f).tobytes(), (what, k, f)


@pytest.mark.parametrize("world", [2, 8])
def test_mesh_on_every_rank_equals_the_single_gpu_mesh(world):
    single = _single(mesh=True)
    ranks = _ranks(world, mesh=True)
    for k, s in enumerate(_scans(4)):
        single.integ.integratePointCloud((s[2], s[3]), s[0], s[1])
        for rk in ranks:
            rk.integ.integratePointCloud((s[2], s[3]), s[0], s[1])
        _exchange(ranks)
        single.mint.generateMesh(True, True)
        for rk in ranks:
            rk.mint.generateMesh(True, True)
            assert rk.mint.last_blocks == single.mint.last_blocks, (k, rk.rank)
            _assert_same_meshes(rk.mesh, single.mesh, f"scan {k} rank {rk.rank}")
    single.mint.generateMesh(False, True)
    for rk in ranks:
        rk.mint.generateMesh(False, True)
        _assert_same_meshes(rk.mesh, single.mesh, f"full mesh rank {rk.rank}")


# ---------------------------------------------------------------- 3. ESDF
ESDF_CONFIGS = {"min_diff_zero": dict(min_diff_m=0.0, multi_queue=1), "ros_default": dict(min_diff_m=1e-3, multi_queue=0)}


def _esdf_compare(esdf, ref, what):
    """Block set and every voxel's flags equal; returns (voxels observed, voxels whose distance differs > 1e-4)."""
    a, b = esdf.blocks(), ref.blocks()
    assert sorted(a) == sorted(b), f"{what}: ESDF block set differs"
    n_obs = n_diff = 0
    for k in b:
        va, vb_ = a[k], b[k]
        for f in ("observed", "hallucinated", "fixed"):
            assert (va[f] == vb_[f]).all(), (what, k, f)
        obs = vb_["observed"] != 0
        n_obs += int(obs.sum())
        n_diff += int((np.abs(va["distance"][obs] - vb_["distance"][obs]) > 1e-4).sum())
    return n_obs, n_diff


@pytest.mark.parametrize("config", list(ESDF_CONFIGS))
@pytest.mark.parametrize("world", [3, 8])
def test_esdf_on_every_rank_matches_the_single_gpu_esdf(world, config):
    voxel, vps, max_d = 0.1, 16, 2.0
    ekw = dict(max_distance_m=max_d, default_distance_m=max_d, min_distance_m=0.2, **ESDF_CONFIGS[config])
    single = _single(esdf=ekw)
    ranks = _ranks(world, esdf=ekw)
    worst = 0.0

    def step(update, incremental):
        nonlocal worst
        befores = [rk.esdf.blocks() for rk in ranks]
        update(single.eint)
        for rk, before in zip(ranks, befores):
            update(rk.eint)
            n_obs, n_diff = _esdf_compare(rk.esdf, single.esdf, f"rank {rk.rank}")
            share = n_diff / max(n_obs, 1)
            worst = max(worst, share)
            rep = fp.counts(fp.fixed_point(rk.esdf.blocks(), voxel, vps, ekw, incremental=incremental,
                                           parents=not incremental, before=before))
            print(world, config, "rank", rk.rank, "incremental" if incremental else "batch", rep,
                  "distance share", n_diff, "/", n_obs)
            if incremental:
                assert rep["a_other"] == 0 and rep["b_other"] == 0 and rep["b_parent_raised"] == 0, rep
            else:
                assert rep["a"] == 0 and rep["b"] == 0 and rep["c"] in (None, 0), rep

    for s in _scans(3):
        single.integ.integratePointCloud((s[2], s[3]), s[0], s[1])
        for rk in ranks:
            rk.integ.integratePointCloud((s[2], s[3]), s[0], s[1])
        _exchange(ranks)
        step(lambda e: e.updateFromTsdfLayer(True), True)
    step(lambda e: e.updateFromTsdfLayerBatch(), False)
    print(world, config, "largest share of observed voxels more than 1e-4 apart:", worst)
    assert worst <= MAX_DISTANCE_SHARE


# ---------------------------------------------------------------- 4. ICP
@pytest.mark.parametrize("world", [3, 8])
def test_icp_against_a_replica_equals_the_single_gpu_map(world):
    scans = list(_scans(4))
    single = _single()
    ranks = _ranks(world)
    for s in scans[:3]:
        single.integ.integratePointCloud((s[2], s[3]), s[0], s[1])
        for rk in ranks:
            rk.integ.integratePointCloud((s[2], s[3]), s[0], s[1])
        _exchange(ranks)
    s = scans[3]
    for k, (dt, yaw) in enumerate(PERTURBATIONS):
        q0, t0 = _perturbed(s, dt, yaw)
        want = vb.ICP(vb.ICPConfig(num_threads=1)).runICP(single.layer, s[0], (q0, t0), seed=7 + k)
        for rk in ranks:
            got = vb.ICP(vb.ICPConfig(num_threads=1)).runICP(rk.layer, s[0], (q0, t0), seed=7 + k)
            assert got[0] == want[0], (rk.rank, got[0], want[0])
            assert got[1][0].tobytes() == want[1][0].tobytes() and got[1][1].tobytes() == want[1][1].tobytes()


# ---------------------------------------------------------------- 5. errors
def _code(excinfo):
    return int(str(excinfo.value).split("(")[1].split(")")[0])


def test_gather_and_upload_errors():
    world = 2
    ranks = _ranks(world)
    s = next(iter(_scans(1)))
    for rk in ranks:
        rk.integ.integratePointCloud((s[2], s[3]), s[0], s[1])
    r0 = ranks[0]
    lay = r0.layer
    bb = lay._block_bytes()
    n = lay.gatherUpdatedDevice(api.UPDATED_MIRROR, owned_only=True)
    assert n > 1
    # cap too small: the count is reported, nothing is copied or cleared
    idx = torch.full((n - 1, 3), -7, dtype=torch.int32, device="cuda")
    vox = torch.zeros((n - 1) * bb, dtype=torch.uint8, device="cuda")
    assert lay.gatherUpdatedDevice(api.UPDATED_MIRROR, api.UPDATED_MIRROR, True, idx, vox) == n
    assert (idx == -7).all() and (vox == 0).all()
    assert lay.gatherUpdatedDevice(api.UPDATED_MIRROR, owned_only=True) == n
    # host and null pointers
    h_idx, h_vox = np.zeros((n, 3), np.int32), np.zeros(n * bb, np.uint8)
    for a, b in ((h_idx.ctypes.data, h_vox.ctypes.data), (0, 0)):
        with pytest.raises(vb.VoxbloxError) as e:
            lay.gatherUpdatedDevice(api.UPDATED_MIRROR, api.UPDATED_MIRROR, True, a, b, cap=n)
        assert _code(e) == 1
        with pytest.raises(vb.VoxbloxError) as e:
            lay.insertBlocksDevice(a, b, m=1)
        assert _code(e) == 1
    assert lay.gatherUpdatedDevice(api.UPDATED_MIRROR, owned_only=True) == n
    before = _layer_state(lay)
    # a block index outside +-2^20, and a block this rank owns: refused before anything is written
    one = torch.zeros(bb, dtype=torch.uint8, device="cuda")
    far = torch.tensor([[(1 << 20) + 1, 0, 0]], dtype=torch.int32, device="cuda")
    assert sharded.block_owner(far.cpu().numpy(), world)[0] == 1
    mine = torch.tensor([[0, 0, 0], [1, 0, 0]], dtype=torch.int32, device="cuda")  # (owners 0 and 1)
    for bad, vox_ in ((far, one), (mine, torch.zeros(2 * bb, dtype=torch.uint8, device="cuda"))):
        with pytest.raises(vb.VoxbloxError) as e:
            lay.insertBlocksDevice(bad, vox_)
        assert _code(e) == 1
    after = _layer_state(lay)
    assert all(x.tobytes() == y.tobytes() for x, y in zip(before, after)), "a refused upload changed the map"
    # the staging buffer of the host paths was never allocated
    assert lay.stagingBytes() == 0


def test_replica_upload_past_the_pool_reports_capacity():
    """A rank whose pool holds its own blocks and half of what it receives: VBX_E_CAPACITY, the pool ends
    full, and every block the upload created holds what was sent for it (DESIGN.md section 9)."""
    world = 2
    scans = list(_scans(2))
    sizing = _ranks(world)
    for s in scans:
        for rk in sizing:
            rk.integ.integratePointCloud((s[2], s[3]), s[0], s[1])
    n0, n1 = (rk.layer.getNumberOfAllocatedBlocks() for rk in sizing)
    assert n1 >= 2
    cap = n0 + n1 // 2
    gather = sharded.LocalAllGather(world)
    small = Rank(0, world, gather, opts=dict(max_blocks=cap, max_updates_per_pass=1 << 22))
    big = Rank(1, world, gather)
    for s in scans:
        for rk in (small, big):
            rk.integ.integratePointCloud((s[2], s[3]), s[0], s[1])
    with ThreadPoolExecutor(2) as ex:
        f_small, f_big = ex.submit(small.sl.exchange), ex.submit(big.sl.exchange)
        assert f_big.result() == n0
        with pytest.raises(vb.VoxbloxError) as e:
            f_small.result()
    assert _code(e) == 3
    assert small.layer.getNumberOfAllocatedBlocks() == cap
    theirs = big.layer.blocks()
    idx = small.layer.getAllAllocatedBlocks()
    got = small.layer.blocks()
    replicas = [tuple(i) for i in idx[~small.owned(idx)].tolist()]
    assert len(replicas) == cap - n0
    for k in replicas:
        assert got[k].tobytes() == theirs[k].tobytes(), k


# ---------------------------------------------------------------- 6. two processes, NCCL
def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _worker(rank, world, port, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        ekw = dict(max_distance_m=2.0, default_distance_m=2.0, min_distance_m=0.2, min_diff_m=0.0, multi_queue=1)
        opts = sharded.shard_options(rank, world, device=rank, **OPTS)
        layer = vb.Layer(0.1, 16, engine_options=opts)
        integ = vb.TsdfIntegratorFactory.create(2, vb.TsdfIntegratorConfig(**CFG), layer)
        esdf = vb.Layer(0.1, 16, voxel_type="esdf")
        eint = vb.EsdfIntegrator(vb.EsdfIntegratorConfig(**ekw), layer, esdf)
        mesh = vb.MeshLayer(layer.block_size())
        mint = vb.MeshIntegrator(vb.MeshIntegratorConfig(), layer, mesh)
        sl = sharded.ShardedLayer(layer)
        for s in _scans():
            integ.integratePointCloud((s[2], s[3]), s[0], s[1])
            sl.exchange()
        staging = layer.stagingBytes()  # (read before the checks below, which download through the host)
        eint.updateFromTsdfLayerBatch()
        mint.generateMesh(False, True)
        idx, vox, _ = _layer_state(layer)
        eb = esdf.blocks()
        ek = sorted(eb)
        flags = np.stack([np.stack([eb[k]["observed"], eb[k]["hallucinated"], eb[k]["fixed"]]) for k in ek])
        mk = mesh.getAllAllocatedMeshes()
        mv = [np.concatenate([m.vertices.view(np.uint8).ravel(), m.normals.view(np.uint8).ravel(),
                              m.colors.ravel()]) for m in (mesh.getMeshPtrByIndex(k) for k in mk.tolist())]
        np.savez(out + f".{rank}.npz", idx=idx, vox=vox.view(np.uint8), staging=staging, ek=np.array(ek, np.int32),
                 flags=flags, mk=mk, mv=np.concatenate(mv) if mv else np.zeros(0, np.uint8))
    finally:
        dist.destroy_process_group()


def test_exchange_over_nccl_world2(tmp_path):
    world = 2
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    ekw = dict(max_distance_m=2.0, default_distance_m=2.0, min_distance_m=0.2, min_diff_m=0.0, multi_queue=1)
    single = _single(esdf=ekw, mesh=True)
    for s in _scans():
        single.integ.integratePointCloud((s[2], s[3]), s[0], s[1])
    single.eint.updateFromTsdfLayerBatch()
    single.mint.generateMesh(False, True)
    ref_idx, ref_vox, _ = _layer_state(single.layer)
    eb = single.esdf.blocks()
    ek = sorted(eb)
    ref_flags = np.stack([np.stack([eb[k]["observed"], eb[k]["hallucinated"], eb[k]["fixed"]]) for k in ek])
    mk = single.mesh.getAllAllocatedMeshes()
    ref_mv = np.concatenate([np.concatenate([m.vertices.view(np.uint8).ravel(), m.normals.view(np.uint8).ravel(),
                                             m.colors.ravel()]) for m in (single.mesh.getMeshPtrByIndex(k)
                                                                          for k in mk.tolist())])
    out = str(tmp_path / "exchange")
    port = _free_port()
    ctx = mp.get_context("spawn")
    procs = [ctx.Process(target=_worker, args=(r, world, port, out)) for r in range(world)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(300)
        assert p.exitcode == 0
    for r in range(world):
        z = np.load(out + f".{r}.npz")
        assert int(z["staging"]) == 0, "a payload passed through the page-locked staging buffer"
        assert z["idx"].tolist() == ref_idx.tolist()
        assert z["vox"].tobytes() == ref_vox.view(np.uint8).tobytes(), f"rank {r} map differs from the single-GPU map"
        assert z["ek"].tolist() == [list(k) for k in ek] and (z["flags"] == ref_flags).all()
        assert z["mk"].tolist() == mk.tolist() and z["mv"].tobytes() == ref_mv.tobytes()
