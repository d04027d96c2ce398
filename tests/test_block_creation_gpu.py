"""-m gpu: a call that runs out of pool slots while it creates blocks -- an upload into the TSDF or the ESDF
layer, or addNewRobotPosition -- leaves the map as a scan that overflows does (test_tsdf_gpu.py's
test_pool_overflow_is_reported_and_does_not_poison_later_calls): the call raises, the blocks it created are
counted and listed and hold what it put there, the pool stays full, no two block indices share a pool slot, no
index stays in the hash without a slot, and the emptied map integrates like the reference again."""
import numpy as np
import pytest

import voxblox_b200 as vb
from oracle import pyoracle as po
from tests.parity import compare_tsdf
from voxblox_b200 import scenes

pytestmark = pytest.mark.gpu

MAX_BLOCKS, VPS = 8, 16
ROBOT = np.array([30.0, -20.0, 5.0], np.float32)  # far from the blocks uploaded first


def _map(max_blocks, with_esdf):
    cfg = vb.TsdfIntegratorConfig(default_truncation_distance=0.4, integrator_threads=1)
    layer = vb.Layer(0.1, VPS, engine_options=vb.EngineOptions(max_blocks=max_blocks))
    integ = vb.TsdfIntegratorFactory.create("merged", cfg, layer)
    esdf = eint = None
    if with_esdf:
        esdf = vb.Layer(0.1, VPS, voxel_type="esdf")
        eint = vb.EsdfIntegrator(vb.EsdfIntegratorConfig(), layer, esdf)
    return layer, integ, esdf, eint


def _payload(dtype, n, seed):
    """n blocks of voxels no two of which are alike."""
    rng = np.random.default_rng(seed)
    v = np.zeros((n, VPS ** 3), dtype)
    v["distance"] = rng.uniform(-0.4, 0.4, v.shape).astype(np.float32)
    if dtype == vb.TSDF_DTYPE:
        v["weight"] = rng.uniform(0.5, 9.0, v.shape).astype(np.float32)
        v["color"] = rng.integers(0, 256, v.shape + (4,), dtype=np.uint8)
    else:
        v["observed"] = 1
        v["parent"] = rng.integers(-3, 4, v.shape + (3,), dtype=np.int32)
    return v


def _row(n, x0):
    return np.array([[x0 + i, 3, -2] for i in range(n)], np.int32)


def _assert_holds(target, want):
    listed = target.getAllAllocatedBlocks()
    got = target.getBlocks(listed)[0]
    for k, i in enumerate(listed.tolist()):
        assert got[k].tobytes() == want[tuple(i)].tobytes(), i


@pytest.mark.parametrize("case", ["tsdf_upload", "esdf_upload", "robot_position"])
def test_pool_overflow_while_creating_blocks(case):
    layer, integ, esdf, eint = _map(MAX_BLOCKS, with_esdf=case != "tsdf_upload")
    target = layer if case == "tsdf_upload" else esdf
    dt = vb.TSDF_DTYPE if target is layer else vb.ESDF_DTYPE
    first = _row(3, 0)
    first_vox = _payload(dt, len(first), 1)
    target.insertBlocks(first, first_vox)
    want = {tuple(i): first_vox[k] for k, i in enumerate(first.tolist())}  # what each block must hold
    if case == "robot_position":
        with pytest.raises(vb.VoxbloxError):
            eint.addNewRobotPosition(ROBOT)
        # the same call with room to spare: what each block it creates holds (the sphere's rules are per voxel)
        _, _, roomy, roomy_int = _map(4096, with_esdf=True)
        roomy_int.addNewRobotPosition(ROBOT)
        tried = roomy.getAllAllocatedBlocks()
        assert len(tried) > MAX_BLOCKS
        tried_vox = roomy.getBlocks(tried)[0]
    else:
        tried = _row(MAX_BLOCKS, 100)  # more new blocks than there are free slots, as many as the pool holds
        tried_vox = _payload(dt, len(tried), 2)
        with pytest.raises(vb.VoxbloxError):
            target.insertBlocks(tried, tried_vox)
    want.update({tuple(i): tried_vox[k] for k, i in enumerate(tried.tolist())})

    n = target.getNumberOfAllocatedBlocks()
    listed = target.getAllAllocatedBlocks()
    assert n <= MAX_BLOCKS and len(listed) == n
    assert {tuple(i) for i in first.tolist()} <= {tuple(i) for i in listed.tolist()}
    # the blocks the call created fill the pool: a block at a new index cannot be stored
    with pytest.raises(vb.VoxbloxError):
        layer.insertBlocks(np.array([[-50, 50, 50]], np.int32), _payload(vb.TSDF_DTYPE, 1, 3))
    assert not layer.hasBlock((-50, 50, 50))
    _assert_holds(target, want)

    # Every index tried, one block per call with a payload of its own: a call either stores its block where
    # that index alone is found, or raises and leaves no block behind.
    keys = np.concatenate([first, tried])
    mine = _payload(dt, len(keys), 4)
    for k, i in enumerate(keys.tolist()):
        try:
            target.insertBlocks(np.array([i], np.int32), mine[k:k + 1])
            stored = True
        except vb.VoxbloxError:
            stored = False
        assert stored == target.hasBlock(i), i
        if stored:
            want[tuple(i)] = mine[k]
    _assert_holds(target, want)

    if esdf is not None:
        esdf.removeAllBlocks()
        assert esdf.getNumberOfAllocatedBlocks() == 0
    layer.removeAllBlocks()
    assert layer.getNumberOfAllocatedBlocks() == 0
    s = scenes.c3_room_sequence(n_scans=1, width=96, height=72)[0]
    few = (s[0][:1], s[1][:1], s[2], s[3])  # one ray: a handful of blocks fits
    integ.integratePointCloud((few[2], few[3]), few[0], few[1])
    omap = po.OracleMap(po.OracleLib("port"), po.TsdfConfig(default_truncation_distance=0.4), 0.1, VPS)
    omap.integrate(2, few)
    rep = compare_tsdf(layer, omap)
    assert rep["blocks_equal"] and rep["n_bit_exact"] == rep["n_voxels"], rep
