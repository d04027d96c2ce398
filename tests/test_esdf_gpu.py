"""-m gpu parity: the device ESDF wavefront against the CPU oracle."""
import numpy as np
import pytest

import voxblox_b200 as vb
from oracle import pyoracle as po
from tests.parity import compare_esdf, compare_tsdf
from voxblox_b200 import scenes

pytestmark = pytest.mark.gpu


def _setup(voxel_size, trunc, ekw):
    cfg = vb.TsdfIntegratorConfig(default_truncation_distance=trunc, integrator_threads=1)
    tsdf = vb.Layer(voxel_size, 16)
    integ = vb.TsdfIntegratorFactory.create("merged", cfg, tsdf)
    esdf = vb.Layer(voxel_size, 16, voxel_type="esdf")
    eint = vb.EsdfIntegrator(vb.EsdfIntegratorConfig(**ekw), tsdf, esdf)
    omap = po.OracleMap(po.OracleLib("port"), po.TsdfConfig(default_truncation_distance=trunc), voxel_size, 16)
    omap.esdf_create(po.EsdfConfig(**ekw))
    return tsdf, integ, esdf, eint, omap


# the reference's own ESDF test configuration (test_sdf_integrators.cc:196-203)
EKW = dict(max_distance_m=4.0, default_distance_m=4.0, min_distance_m=0.2, min_diff_m=0.0, multi_queue=1)


def test_esdf_batch_matches_oracle():
    scans = scenes.c3_room_sequence(n_scans=4, width=160, height=120)
    tsdf, integ, esdf, eint, omap = _setup(0.1, 0.4, EKW)
    for s in scans:
        integ.integratePointCloud((s[2], s[3]), s[0], s[1])
        omap.integrate(2, s, order=po.ORDER_REFERENCE)
    assert compare_tsdf(tsdf, omap)["max_rel_err"] == 0.0
    eint.updateFromTsdfLayerBatch()
    omap.esdf_update(batch=True)
    rep = compare_esdf(esdf, omap, 4.0)
    print(rep, eint.counters())
    assert rep["blocks_equal"] and rep["observed_equal"] and rep["fixed_equal"], rep
    assert rep["flag_bytes_clean"] and rep["in_queue_gpu"] == 0, rep
    # Same-sign propagation converges to an order-independent fixed point (bit-exact); where a
    # free voxel touches a voxel of the opposite sign the reference ASSIGNS sign*dist in queue
    # order (esdf_integrator.cc:458-488) and no parallel order can reproduce it -- bound it.
    assert rep["n_bit_exact"] >= 0.93 * rep["voxels_observed"], rep
    assert rep["rmse"] < 0.1 * 0.1, rep
    assert rep["max_abs_err"] <= 2 * 0.1 * 3 ** 0.5, rep


def _wall_scans():
    """A wall seen from three poses: no thin structures, so no opposite-sign neighbours."""
    dirs = scenes.pinhole_dirs(160, 120, 131.25, 131.25, 80.0, 60.0)
    prims = [scenes.Plane((0.0, 0.0, 1.0), 3.0)]
    out = []
    for k in range(3):
        q = scenes.quat_from_rpy(0.013 + 0.05 * k, -0.021 - 0.04 * k, 0.017)
        t = np.array([0.013 + 0.3 * k, 0.021 - 0.2 * k, 0.017 + 0.1 * k])
        out.append(scenes.render(prims, dirs, q, t))
    return out


def test_esdf_batch_exact_without_sign_conflicts():
    tsdf, integ, esdf, eint, omap = _setup(0.1, 0.4, EKW)
    for s in _wall_scans():
        integ.integratePointCloud((s[2], s[3]), s[0], s[1])
        omap.integrate(2, s, order=po.ORDER_REFERENCE)
    eint.updateFromTsdfLayerBatch()
    omap.esdf_update(batch=True)
    rep = compare_esdf(esdf, omap, 4.0)
    print(rep, eint.counters())
    assert rep["blocks_equal"] and rep["observed_equal"] and rep["fixed_equal"], rep
    assert rep["n_over_1e-4"] <= 0.002 * rep["voxels_observed"], rep


def test_esdf_incremental_tracks_oracle():
    scans = scenes.c3_room_sequence(n_scans=4, width=160, height=120)
    tsdf, integ, esdf, eint, omap = _setup(0.1, 0.4, EKW)
    for s in scans:
        integ.integratePointCloud((s[2], s[3]), s[0], s[1])
        omap.integrate(2, s, order=po.ORDER_REFERENCE)
        eint.updateFromTsdfLayer(True)
        omap.esdf_update(batch=False, clear_updated_flag=True)
        rep = compare_esdf(esdf, omap, 4.0)
        print(rep, eint.counters())
        assert rep["blocks_equal"] and rep["observed_equal"] and rep["fixed_equal"], rep
    assert len(tsdf.getAllUpdatedBlocks(2)) == 0  # kEsdf bits were cleared
    frac_bad = rep["n_over_1e-4"] / max(1, rep["voxels_observed"])
    # the reference's own incremental-vs-batch criterion is statistical (test_sdf_integrators.cc:261-270)
    assert rep["rmse"] < 4.0 * 0.1, rep
    assert frac_bad < 0.06, rep  # same order-dependent sign-conflict voxels as in the batch test


def test_update_from_tsdf_blocks_and_setters():
    """updateFromTsdfBlocks(list, incremental=False) on a subset of blocks (missing and repeated
    indices included), then setEsdfMaxDistance / setFullEuclidean followed by a batch update
    (esdf_integrator.h:111-112,139-149)."""
    tsdf, integ, esdf, eint, omap = _setup(0.1, 0.4, EKW)
    for s in _wall_scans():
        integ.integratePointCloud((s[2], s[3]), s[0], s[1])
        omap.integrate(2, s, order=po.ORDER_REFERENCE)
    blocks = tsdf.getAllAllocatedBlocks()
    subset = np.concatenate([blocks[::2], blocks[:1], np.array([[900, 900, 900]], np.int32)])
    eint.updateFromTsdfBlocks(subset)
    omap.esdf_update_blocks(np.concatenate([blocks[::2], np.array([[900, 900, 900]], np.int32)]))
    rep = compare_esdf(esdf, omap, 4.0)
    print(rep)
    assert rep["blocks_equal"] and rep["observed_equal"] and rep["fixed_equal"], rep
    assert rep["n_bit_exact"] >= 0.995 * rep["voxels_observed"], rep
    # setters behave like the reference's
    assert eint.getEsdfMaxDistance() == pytest.approx(4.0)
    eint.setEsdfMaxDistance(5.0)
    omap.esdf_set_max_distance(5.0)
    assert eint.getEsdfMaxDistance() == pytest.approx(5.0)
    assert eint._config().default_distance_m == pytest.approx(5.0)   # follows upwards, h:142-144
    eint.setFullEuclidean(True)
    omap.esdf_set_full_euclidean(True)
    assert eint.getFullEuclidean() is True
    eint.updateFromTsdfLayerBatch()
    omap.esdf_update(batch=True)
    rep = compare_esdf(esdf, omap, 5.0)
    print("full Euclidean", rep)
    assert rep["blocks_equal"] and rep["observed_equal"] and rep["fixed_equal"] and rep["hallucinated_equal"], rep
    assert rep["rmse"] <= 0.3 * 0.1, rep   # (the reference's own full-Euclidean result depends on its pop order)
    eint.setFullEuclidean(False)
    omap.esdf_set_full_euclidean(False)
    eint.updateFromTsdfLayerBatch()
    omap.esdf_update(batch=True)
    rep = compare_esdf(esdf, omap, 5.0)
    print(rep)
    assert rep["blocks_equal"] and rep["observed_equal"] and rep["fixed_equal"], rep
    assert rep["n_bit_exact"] >= 0.995 * rep["voxels_observed"], rep


# test_clear_spheres.cc:118-129 at a smaller occupied radius
EKW_SPHERES = dict(max_distance_m=2.0, default_distance_m=2.0, min_distance_m=0.2, min_diff_m=0.0,
                   clear_sphere_radius=1.0, occupied_sphere_radius=2.5)


def _esdf_bytes_equal(esdf, omap):
    gi, oi = esdf.getAllAllocatedBlocks(), omap.block_indices(1)
    if gi.shape != oi.shape or not (gi == oi).all():
        return False
    gv, _ = esdf.getBlocks(gi)
    return all(gv[k].tobytes() == omap.block(i, 1)[0].tobytes() for k, i in enumerate(oi))


def test_add_new_robot_position_matches_oracle():
    """EsdfIntegrator::addNewRobotPosition (esdf_integrator.cc:25-92) on the device, driven like the
    reference's test_clear_spheres.cc:107-165: sphere, scan, incremental update, twice."""
    scans = scenes.c3_room_sequence(n_scans=2, width=160, height=120)
    tsdf, integ, esdf, eint, omap = _setup(0.1, 0.4, EKW_SPHERES)
    # 1. the spheres alone, on an empty map: deterministic -> every voxel bit-identical, and the
    #    TSDF layer still holds no block (the sphere allocates ESDF blocks only)
    eint.addNewRobotPosition(scans[0][3])
    omap.esdf_add_robot_position(scans[0][3])
    c = eint.counters()
    print("sphere counters", c)
    assert _esdf_bytes_equal(esdf, omap)
    assert len(tsdf.getAllAllocatedBlocks()) == 0 and tsdf.getNumberOfAllocatedBlocks() == 0
    assert len(esdf.getAllAllocatedBlocks()) == c["blocks"] > 0
    for k, s in enumerate(scans):
        if k > 0:
            eint.addNewRobotPosition(s[3])
            omap.esdf_add_robot_position(s[3])
        integ.integratePointCloud((s[2], s[3]), s[0], s[1])
        omap.integrate(2, s, order=po.ORDER_REFERENCE)
        assert compare_tsdf(tsdf, omap)["max_rel_err"] == 0.0
        eint.updateFromTsdfLayer(True)
        omap.esdf_update(batch=False, clear_updated_flag=True)
        rep = compare_esdf(esdf, omap, 2.0)
        print(k, rep, eint.counters())
        assert rep["blocks_equal"] and rep["observed_equal"] and rep["fixed_equal"], rep
        assert rep["hallucinated_equal"] and rep["flag_bytes_clean"] and rep["in_queue_gpu"] == 0, rep
        assert rep["rmse"] < 0.1, rep
        assert rep["n_over_1e-4"] < 0.08 * rep["voxels_observed"], rep
    # the reference test's own criteria (test_clear_spheres.cc:171-203) on the device layers
    ti = tsdf.getAllAllocatedBlocks()
    tv, _ = tsdf.getBlocks(ti)
    ev, _ = esdf.getBlocks(ti)          # ASSERT_TRUE(esdf_layer.hasBlock(block_index))
    unobs = tv["weight"] < 1e-6
    assert (ev["hallucinated"][unobs & (ev["observed"] != 0)] != 0).all()
    band = (tv["weight"] > 1e-6) & (np.abs(tv["distance"]) <= 0.2)
    assert (ev["observed"][band] != 0).all() and (ev["hallucinated"][band] == 0).all()
    assert (np.sign(tv["distance"][band]) == np.sign(ev["distance"][band])).all()
    assert np.abs(tv["distance"][band] - ev["distance"][band]).max() <= 1e-3


def test_esdf_clear_drops_robot_position_queue():
    """EsdfIntegrator::clear() (esdf_integrator.h:135-140): nothing queued by addNewRobotPosition
    reaches the next update."""
    scans = scenes.c3_room_sequence(n_scans=1, width=160, height=120)
    tsdf, integ, esdf, eint, omap = _setup(0.1, 0.4, EKW_SPHERES)
    s = scans[0]
    integ.integratePointCloud((s[2], s[3]), s[0], s[1])
    eint.updateFromTsdfLayer(True)
    eint.addNewRobotPosition(s[3])
    assert eint.counters()["relaxations"] > 0      # slot [5] after the sphere call: open_ entries queued
    eint.clear()
    eint.updateFromTsdfLayer(True)
    c = eint.counters()
    assert c["blocks"] == 0 and c["relaxations"] == 0 and c["raised_voxels"] == 0, c


@pytest.mark.parametrize("vps", [8, 4])
def test_esdf_other_block_sizes(vps):
    """voxels_per_side 8 and 4: the propagation kernel stages 6 KiB + 10 KiB (768 B + 1280 B) slabs with the same
    TMA bulk copies as the 48 KiB + 80 KiB ones of the default block size."""
    cfg = vb.TsdfIntegratorConfig(default_truncation_distance=0.4, integrator_threads=1)
    tsdf = vb.Layer(0.1, vps)
    integ = vb.TsdfIntegratorFactory.create("merged", cfg, tsdf)
    esdf = vb.Layer(0.1, vps, voxel_type="esdf")
    eint = vb.EsdfIntegrator(vb.EsdfIntegratorConfig(**EKW), tsdf, esdf)
    omap = po.OracleMap(po.OracleLib("port"), po.TsdfConfig(default_truncation_distance=0.4), 0.1, vps)
    omap.esdf_create(po.EsdfConfig(**EKW))
    for s in _wall_scans():
        integ.integratePointCloud((s[2], s[3]), s[0], s[1])
        omap.integrate(2, s, order=po.ORDER_REFERENCE)
        eint.updateFromTsdfLayer(True)
        omap.esdf_update(batch=False, clear_updated_flag=True)
    gi, oi = esdf.getAllAllocatedBlocks(), omap.block_indices(1)
    assert gi.shape == oi.shape and (gi == oi).all()
    gv, _ = esdf.getBlocks(gi)
    ov = np.stack([omap.block(i, 1)[0] for i in oi])
    obs = ov["observed"] != 0
    assert ((gv["observed"] != 0) == obs).all() and (gv["fixed"][obs] == ov["fixed"][obs]).all()
    exact = (gv["distance"][obs] == ov["distance"][obs]).mean()
    print("vps", vps, "observed", int(obs.sum()), "bit-exact fraction", exact)
    assert exact >= 0.995
