"""-m gpu: one view of which pool slots hold a block of each layer.  The TSDF and the ESDF layer share
pool slots, so a slot may hold both blocks, the ESDF block only (ESDF uploads, robot-position spheres, a
removed TSDF block), the TSDF block only (a removed ESDF block) or neither; every listing, download,
mirror, mesh and removal must agree on which blocks each layer holds."""
import numpy as np
import pytest

import voxblox_b200 as vb
from voxblox_b200 import scenes

pytestmark = pytest.mark.gpu

VPS = 16
FAR = [[40, -40, 7], [41, -40, 7], [-30, 25, -3]]  # ESDF uploads at indices no scan reaches


def _keys(idx):
    return [tuple(int(v) for v in i) for i in np.asarray(idx).reshape(-1, 3)]


def _esdf_vox(n, d):
    vox = np.zeros((n, VPS ** 3), vb.ESDF_DTYPE)
    vox["distance"] = d
    vox["observed"] = 1
    return vox


def _clear_bits(layer, mask):
    """vbx_clear_updated with a raw bit mask (Layer.clearUpdated takes one bit)."""
    ctx = layer._bound()
    ctx.check(ctx.lib.vbx_clear_updated(ctx.handle, layer._layer_id, mask), "vbx_clear_updated")


def _snapshot(layer):
    """{index: (payload bytes, reported bits)} through the listing + per-block download path."""
    idx = layer.getAllAllocatedBlocks()
    vox, upd = layer.getBlocks(idx)
    return {k: (vox[i].tobytes(), int(upd[i])) for i, k in enumerate(_keys(idx))}


def _mixed_map():
    """A map that holds every kind of slot at once.  Returns the layers, the integrators and the index
    sets each kind was built from."""
    cfg = vb.TsdfIntegratorConfig(default_truncation_distance=0.4, integrator_threads=1)
    opts = vb.EngineOptions(max_blocks=8192, max_updates_per_pass=1 << 22)
    layer = vb.Layer(0.1, VPS, engine_options=opts)
    integ = vb.TsdfIntegratorFactory.create("merged", cfg, layer)
    esdf = vb.Layer(0.1, VPS, voxel_type="esdf")
    eint = vb.EsdfIntegrator(vb.EsdfIntegratorConfig(min_distance_m=0.2, clear_sphere_radius=0.5,
                                                     occupied_sphere_radius=1.0), layer, esdf)
    first = [[-60, 60, 60]]
    layer.insertBlocks(np.array(first, np.int32), np.zeros((1, VPS ** 3), vb.TSDF_DTYPE))  # the lowest slot
    for s in scenes.c3_room_sequence(n_scans=2, width=128, height=96):
        integ.integratePointCloud((s[2], s[3]), s[0], s[1])
    eint.updateFromTsdfLayer(True)  # an ESDF block in every slot a scan touched (the uploaded one has no kEsdf bit)
    both = esdf.getAllAllocatedBlocks()
    assert set(_keys(layer.getAllAllocatedBlocks())) == set(_keys(both)) | set(_keys(first))
    esdf.insertBlocks(np.array(FAR, np.int32), _esdf_vox(len(FAR), 1.25))
    before = set(_keys(esdf.getAllAllocatedBlocks()))
    eint.addNewRobotPosition([30.0, 30.0, 30.0])
    sphere = sorted(set(_keys(esdf.getAllAllocatedBlocks())) - before)
    assert sphere and not set(sphere) & set(_keys(both))
    tsdf_gone = both[1::4]  # TSDF removed, ESDF stays
    esdf_gone = both[2::4]  # ESDF removed, TSDF stays
    layer.removeBlocks(tsdf_gone)
    esdf.removeBlocks(esdf_gone)
    last = [[61, -61, 61]]
    layer.insertBlocks(np.array(last, np.int32), np.zeros((1, VPS ** 3), vb.TSDF_DTYPE))  # the highest slot
    sets = dict(both=set(_keys(both)) - set(_keys(tsdf_gone)) - set(_keys(esdf_gone)),
                esdf_only=set(_keys(FAR)) | set(sphere) | set(_keys(tsdf_gone)),
                tsdf_only=set(_keys(esdf_gone)) | set(_keys(first)) | set(_keys(last)),
                first=_keys(first)[0], last=_keys(last)[0], sphere=sphere)
    return layer, integ, esdf, eint, sets


def _members_agree(layer, want, others):
    """Block count, listing, mirror, serialisation and per-block download all give the layer's set `want`;
    the download rejects every index in `others`."""
    idx = layer.getAllAllocatedBlocks()
    assert set(_keys(idx)) == want and len(idx) == len(want)
    assert layer.getNumberOfAllocatedBlocks() == len(want)
    midx, mvox, mupd = layer.mirrorUpdated(0, 0)
    sidx, _, supd = layer.serializeUpdated(0, 0)
    assert (midx == idx).all() and (sidx == idx).all()
    vox, upd = layer.getBlocks(idx)
    assert vox.tobytes() == mvox.tobytes() and (upd == mupd).all() and (upd == supd).all()
    for k in sorted(others):
        with pytest.raises(vb.VoxbloxError):
            layer.getBlocks(np.array([k], np.int32))


def test_mixed_map_layers_agree():
    layer, _, esdf, eint, sets = _mixed_map()
    tsdf_set = sets["both"] | sets["tsdf_only"]
    esdf_set = sets["both"] | sets["esdf_only"]
    _members_agree(layer, tsdf_set, sets["esdf_only"])
    _members_agree(esdf, esdf_set, sets["tsdf_only"])
    got, _ = esdf.getBlocks(np.array(FAR, np.int32))
    assert (got["distance"] == 1.25).all()
    # the mesher reads the TSDF layer only
    mesh_layer = vb.MeshLayer(layer.block_size())
    vb.MeshIntegrator(vb.MeshIntegratorConfig(), layer, mesh_layer).generateMesh(False, False)
    meshes = set(_keys(mesh_layer.getAllAllocatedMeshes()))
    assert meshes <= tsdf_set and not meshes & sets["esdf_only"]
    # updateFromTsdfBlocks skips indices without a TSDF block (esdf_integrator.cc:137-141)
    eint.clear()
    esdf_before, tsdf_before = _snapshot(esdf), _snapshot(layer)
    eint.updateFromTsdfBlocks(np.array(sorted(sets["esdf_only"]), np.int32), incremental=False)
    assert eint.counters()["blocks"] == 0
    assert _snapshot(esdf) == esdf_before and _snapshot(layer) == tsdf_before


def test_update_masks_and_clears():
    layer, integ, esdf, eint, sets = _mixed_map()
    tsdf_set = sets["both"] | sets["tsdf_only"]
    # every flag byte of the TSDF layer to 0 (the mirror clear takes every bit a caller may clear)
    layer.mirrorUpdated(0, 0xFF)
    assert all(u == 0 for _, u in _snapshot(layer).values())
    assert set(_keys(layer.getAllAllocatedBlocks())) == tsdf_set
    # a scan sets the three reported bits and the mirror mark of the blocks it touches
    s = scenes.c3_room_sequence(n_scans=3, width=128, height=96)[2]
    integ.integratePointCloud((s[2], s[3]), s[0], s[1])
    snap = _snapshot(layer)
    touched = {k for k, (_, u) in snap.items() if u == 7}
    assert touched and all(u in (0, 7) for _, u in snap.values())
    tsdf_set = set(snap)  # (the scan may have turned ESDF-only slots into TSDF blocks)
    assert not tsdf_set & (set(_keys(FAR)) | set(sets["sphere"]))
    # re-uploading a block with given bits sets them and clears its mirror mark
    keys = sorted(snap)
    rewrite = keys[::3]
    bits = np.array([i % 8 for i in range(len(rewrite))], np.uint8)
    vox, _ = layer.getBlocks(np.array(rewrite, np.int32))
    layer.insertBlocks(np.array(rewrite, np.int32), vox, bits)
    want_bits = {k: (7 if k in touched else 0) for k in keys}
    want_bits.update({k: int(b) for k, b in zip(rewrite, bits)})
    mirror = touched - set(rewrite)
    assert {k: u for k, (_, u) in _snapshot(layer).items()} == want_bits
    for mask in range(1, 16):
        listed = set(_keys(layer._list(mask)))
        assert listed == {k for k in keys if want_bits[k] & mask & 7}, mask
        midx, _, mupd = layer.mirrorUpdated(mask, 0)
        want = {k for k in keys if (want_bits[k] & mask) or (mask & 8 and k in mirror)}
        assert set(_keys(midx)) == want, mask
        assert [int(u) for u in mupd] == [want_bits[k] for k in _keys(midx)], mask
    # clearing every bit, or the ESDF integrator's state, keeps the ESDF-only slots out of the TSDF layer
    _clear_bits(layer, 0xFF)
    _clear_bits(esdf, 0xFF)
    eint.clear()
    assert set(_keys(layer.getAllAllocatedBlocks())) == tsdf_set
    assert layer.getNumberOfAllocatedBlocks() == len(tsdf_set)
    assert set(_keys(esdf.getAllAllocatedBlocks())) == sets["both"] | sets["esdf_only"]
    assert all(u == 0 for _, u in _snapshot(layer).values())


def test_removal_keeps_both_layers():
    layer, integ, esdf, _, sets = _mixed_map()
    tsdf_snap, esdf_snap = _snapshot(layer), _snapshot(esdf)
    both = sorted(sets["both"])
    missing = [[500, 500, 500], [-500, 3, 9]]
    tsdf_batch = ([list(sets["last"]), list(sets["first"])] + [list(k) for k in sorted(sets["esdf_only"])] +
                  [list(k) for k in both[::3]] + missing + [list(k) for k in both[::6]] + [list(sets["last"])])
    esdf_batch = [list(k) for k in sorted(sets["esdf_only"])] + [list(k) for k in both[1::3]] + missing
    steps = [(layer, tsdf_batch[: len(tsdf_batch) // 2]), (esdf, esdf_batch[::2]),
             (layer, tsdf_batch[len(tsdf_batch) // 2:]), (esdf, esdf_batch[1::2] + esdf_batch[:3])]
    for which, batch in steps:
        gone = set(_keys(batch))
        if which is layer:
            tsdf_snap = {k: v for k, v in tsdf_snap.items() if k not in gone}
        else:
            esdf_snap = {k: v for k, v in esdf_snap.items() if k not in gone}
        which.removeBlocks(np.array(batch, np.int32))
        assert _snapshot(layer) == tsdf_snap
        assert _snapshot(esdf) == esdf_snap
        assert layer.getNumberOfAllocatedBlocks() == len(tsdf_snap)
        assert esdf.getNumberOfAllocatedBlocks() == len(esdf_snap)
    # the freed slots read as new blocks: what a scan re-creates equals a fresh map's blocks
    s = scenes.c3_room_sequence(n_scans=3, width=128, height=96)[2]
    integ.integratePointCloud((s[2], s[3]), s[0], s[1])
    cfg = vb.TsdfIntegratorConfig(default_truncation_distance=0.4, integrator_threads=1)
    fresh = vb.Layer(0.1, VPS)
    vb.TsdfIntegratorFactory.create("merged", cfg, fresh).integratePointCloud((s[2], s[3]), s[0], s[1])
    got, want = _snapshot(layer), _snapshot(fresh)
    recreated = [k for k in want if k not in tsdf_snap]
    assert recreated
    for k in recreated:
        assert got[k] == want[k], k


def test_remove_more_than_a_thousand_blocks():
    cfg = vb.TsdfIntegratorConfig(default_truncation_distance=0.4)
    layer = vb.Layer(0.1, VPS, engine_options=vb.EngineOptions(max_blocks=4096, max_updates_per_pass=1 << 20))
    vb.TsdfIntegratorFactory.create("simple", cfg, layer)
    esdf = vb.Layer(0.1, VPS, voxel_type="esdf")
    vb.EsdfIntegrator(vb.EsdfIntegratorConfig(), layer, esdf)
    g = np.stack(np.meshgrid(np.arange(16), np.arange(16), np.arange(8), indexing="ij"), -1).reshape(-1, 3)
    idx = (g - 5).astype(np.int32)
    rng = np.random.default_rng(7)
    vox = np.zeros((len(idx), VPS ** 3), vb.TSDF_DTYPE)
    vox["distance"] = rng.standard_normal(vox.shape).astype(np.float32)
    vox["weight"] = rng.random(vox.shape).astype(np.float32)
    layer.insertBlocks(idx, vox, (np.arange(len(idx)) % 8).astype(np.uint8))
    esdf.insertBlocks(idx[::5], _esdf_vox(len(idx[::5]), 0.5))
    tsdf_snap, esdf_snap = _snapshot(layer), _snapshot(esdf)
    kill = idx[rng.permutation(len(idx))[:1500]]
    assert len(kill) > 1000
    layer.removeBlocks(kill)
    gone = set(_keys(kill))
    assert _snapshot(layer) == {k: v for k, v in tsdf_snap.items() if k not in gone}
    assert _snapshot(esdf) == esdf_snap
    assert layer.getNumberOfAllocatedBlocks() == len(idx) - 1500
