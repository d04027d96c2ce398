"""-m gpu: every voxel of the device ESDF held to the wavefront's fixed point (tests/esdf_fixed_point.py), and
to a float64 shortest-path reference, in quasi-Euclidean mode.

What the device claims does not depend on the order in which it visited voxels, so it is checked exactly:
 * a batch update (fresh layer; over a layer that already holds values -- updateFromTsdfLayerBatch starts with
   esdf_layer_->removeAllBlocks(), esdf_integrator.cc:95, so it rewrites every voxel like a fresh one; or
   updateFromTsdfBlocks on a subset of the blocks of a fresh layer, non-incremental): no rule can still fire (a),
   every value is justified (b), every parent is the first justifier in table order (c, min_diff 0), and
   the values lie at or under the same-sign least fixed point (Dijkstra) and on it where the mixed-sign rule
   cannot reach: zero exceptions;
 * incremental updates (after every scan, and a raise that re-observes the surface as free space): the
   reference's own rules leave exceptions (the unscaled seed step, cc:498-530; sources an update never
   queues; values it does not re-derive).  Each is a class named by a rule on the output
   (esdf_fixed_point.CLASSES), counted on both sides; the device has none outside the named classes, none
   left behind by a raise (a child whose parent rose keeps its old value), and at most as many mixed-sign
   ones as the reference; the other classes are printed.  Incremental kinds include a non-incremental
   updateFromTsdfBlocks over a populated layer, whose observed voxels go through the lower / raise / keep
   branches of the classification (cc:201-282).
The reference side is the reference's own EsdfIntegrator (oracle/_ref) where it was built, else the
restatement held to its recorded digests (tests/golden/reference_pins.py).  Every case prints its counts."""
import numpy as np
import pytest

import voxblox_b200 as vb
from oracle import pyoracle as po
from tests import esdf_fixed_point as fp
from tests import test_esdf_reference_gpu as te
from tests.test_esdf_gpu import _wall_scans
from tests.test_esdf_options_gpu import _freespace_scan
from tests.golden import reference_pins as pins

pytestmark = pytest.mark.gpu


# scene -> (voxel size, truncation, voxels per side, max_distance_m, scans, Dijkstra reference affordable)
SCENES = {
    "wall": (0.1, 0.4, 16, 4.0, _wall_scans, True),
    "room_small": (0.1, 0.4, 16, 2.0, te.ROOM_SMALL["scans"], True),
    "room_small_vps8": (0.1, 0.4, 8, 2.0, te.ROOM_SMALL["scans"], True),
    "room_small_vps4": (0.1, 0.4, 4, 2.0, te.ROOM_SMALL["scans"], True),
    "room_full_640x480": (0.05, 0.2, 16, 2.0, te.ROOM_FULL["scans"], False),
    "cylinder_0.2": (0.2, 0.8, 16, 4.0, te._gt_scans, True),
    "cylinder_0.1": (0.1, 0.4, 16, 4.0, te._gt_scans, False),
}
CONFIGS = {"min_diff_zero": dict(min_diff_m=0.0, multi_queue=1), "ros_default": dict(min_diff_m=1e-3, multi_queue=0)}
BATCH_KINDS = ("batch", "batch_over", "blocks")
INCREMENTAL_KINDS = ("incremental", "raise", "blocks_over")
KEYS = [f"{k}/{c}/{s}" for k in BATCH_KINDS + INCREMENTAL_KINDS for c in CONFIGS for s in SCENES]
PIN_KEYS = KEYS


def _case(key):
    kind, config, scene = key.split("/")
    voxel, trunc, vps, max_d, scans, dij = SCENES[scene]
    ekw = dict(max_distance_m=max_d, default_distance_m=max_d, min_distance_m=trunc / 2, **CONFIGS[config])
    return kind, voxel, trunc, vps, ekw, scans, dij


def _drive(key, scans, integrate, update, update_blocks, tsdf_blocks, esdf_blocks):
    """One case on either side.  Returns the checked updates as (incremental, before, after) ESDF block sets."""
    kind = key.split("/")[0]
    out = []

    def checked(fn, incremental):
        before = esdf_blocks()
        fn()
        out.append((incremental, before, esdf_blocks()))

    if kind in ("batch", "blocks"):
        for s in scans:
            integrate(s, False)
        if kind == "batch":
            checked(lambda: update(True), False)
        else:
            checked(lambda: update_blocks(tsdf_blocks()[::2]), False)
    elif kind == "batch_over":
        for s in scans:
            integrate(s, False)
            update(False)
        checked(lambda: update(True), False)
    elif kind == "incremental":
        for s in scans:
            integrate(s, False)
            checked(lambda: update(False), True)
    elif kind == "blocks_over":
        # non-incremental updateFromTsdfBlocks over a populated layer: its observed voxels go through the lower,
        # raise and keep branches of the classification (cc:201-282) instead of being rewritten
        for s in scans[:-1]:
            integrate(s, False)
            update(False)
        integrate(scans[-1], False)
        checked(lambda: update_blocks(tsdf_blocks()[::2]), True)
    elif kind == "raise":
        for s in scans:
            integrate(s, False)
            update(False)
        for _ in range(2):
            integrate(_freespace_scan(scans[-1]), True)
            checked(lambda: update(False), True)
    else:
        raise KeyError(key)
    return out


def reference_side(key, lib):
    """(checked updates, digest of the ESDF layer after each and of the final TSDF layer) of the oracle."""
    kind, voxel, trunc, vps, ekw, scans, _ = _case(key)
    omap = po.OracleMap(lib, po.TsdfConfig(default_truncation_distance=trunc, integrator_threads=1), voxel, vps)
    omap.esdf_create(po.EsdfConfig(**ekw))
    steps = _drive(key, scans(), lambda s, free: omap.integrate(2, s, freespace=free),
                   lambda batch: omap.esdf_update(batch=batch, clear_updated_flag=True),
                   lambda idx: omap.esdf_update_blocks(idx), lambda: omap.block_indices(0), lambda: omap.blocks(1))
    h = pins.map_digest(omap, (po.LAYER_TSDF,))
    for _, _, after in steps:
        for i in sorted(after):
            h += pins.array_digest(np.array(i, np.int32), after[i])
    return steps, pins.array_digest(np.frombuffer(h.encode(), np.uint8))


def device_side(key):
    kind, voxel, trunc, vps, ekw, scans, _ = _case(key)
    cfg = vb.TsdfIntegratorConfig(default_truncation_distance=trunc, integrator_threads=1)
    tsdf = vb.Layer(voxel, vps)
    integ = vb.TsdfIntegratorFactory.create("merged", cfg, tsdf)
    esdf = vb.Layer(voxel, vps, voxel_type="esdf")
    eint = vb.EsdfIntegrator(vb.EsdfIntegratorConfig(**ekw), tsdf, esdf)
    return _drive(key, scans(), lambda s, free: integ.integratePointCloud((s[2], s[3]), s[0], s[1], freespace_points=free),
                  lambda batch: eint.updateFromTsdfLayerBatch() if batch else eint.updateFromTsdfLayer(True),
                  lambda idx: eint.updateFromTsdfBlocks(idx), tsdf.getAllAllocatedBlocks, esdf.blocks)


def _reports(steps, key):
    kind, voxel, _, vps, ekw, _, dij = _case(key)
    reps = []
    for incremental, before, after in steps:
        rep = fp.counts(fp.fixed_point(after, voxel, vps, ekw, incremental=incremental, parents=not incremental,
                                       before=before))
        if not incremental and dij:
            rep.update({f"dijkstra_{k}": v for k, v in fp.counts(fp.dijkstra_check(after, voxel, vps, ekw)).items()})
        reps.append(rep)
    return reps


@pytest.mark.parametrize("key", KEYS)
def test_esdf_fixed_point(key):
    ref_steps, digest = reference_side(key, pins.lib())
    pins.check(f"esdf_fixed_point/{key}", digest)
    dev, ref = _reports(device_side(key), key), _reports(ref_steps, key)
    for k, (d, r) in enumerate(zip(dev, ref)):
        print(key, "update", k, "\n  device   ", d, "\n  reference", r)
    assert len(dev) == len(ref)
    if key.split("/")[0] in BATCH_KINDS:
        for d in dev:
            assert d["a"] == 0 and d["b"] == 0, d
            assert d["c"] in (None, 0), d
            assert d.get("dijkstra_over", 0) == 0 and d.get("dijkstra_under", 0) == 0, d
    else:
        for d in dev:
            assert d["a_other"] == 0 and d["b_other"] == 0, d
            # the device's raise resets every voxel whose parent points at a raised one
            assert d["b_parent_raised"] == 0, d
        total = {c: (sum(d[c] for d in dev), sum(r[c] for r in ref)) for c in fp.CLASSES}
        print(key, "classes (device, reference):", total)
        # the device keeps the candidate nearest the surface where the reference assigns in pop order
        assert total["a_mixed"][0] <= total["a_mixed"][1], total
        # a_seed, a_stale_source, b_parent_across and b_stale depend on which voxels an update re-derives, which
        # follows each side's parent tree (first justifier against last writer); they are printed, not bounded
        # (measured: the device's b_stale exceeds the reference's on the cylinder scenes, DESIGN.md section 6)
