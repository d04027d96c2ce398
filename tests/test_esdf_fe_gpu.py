"""-m gpu: every full-Euclidean ESDF voxel of the device held to the wavefront's fixed point, its parent roots and a
float64 Euclidean reference (tests/esdf_fe_check.py), beside the reference's own EsdfIntegrator (oracle/_ref) where
that library exists, else the restatement held to its recorded digests (tests/golden/reference_pins.py).

 * Synthetic TSDF layers (inserted block by block on both sides, weight 1, fixed set exactly as intended): one fixed
   voxel in a cube of free voxels across negative block indices at voxels_per_side 16, 4 and 1 (at 1 every step
   crosses a block), outside and mirrored inside (fixed at -0.0); every reached voxel equals |d_f| + vs * |v - f|
   within the telescoping tolerance on both sides.  Two fixed voxels, an axis-aligned and a tilted plane: (a) and (r)
   exact, the distance to the float64 EDT measured on both sides.  A hairpin path, whose way back brings every
   candidate nearer the fixed voxel (a negative step): those voxels stay unreached and the layer is the reference's
   bit for bit.  A strip of blocks with a chain 512 voxels long: the parent code's range [-512, 511], both ends.
 * The room and cylinder scenes of test_esdf_options_gpu.py (batch, incremental with setFullEuclidean(true) switched
   on mid-sequence, a raise), min_diff 0 with multi_queue and the ROS defaults, room_small also at voxels_per_side
   8 and 4.  Batch: zero (a) exceptions and every root fixed; (t) and the distance to the EDT against the
   reference's, with measured margins.  Incremental: no (a) exception outside the named classes, no more
   mixed-sign ones than the reference, and children left rooted through a raised voxel bounded by the reference's.
Every case prints its counts on both sides."""
import numpy as np
import pytest

import voxblox_b200 as vb
from oracle import pyoracle as po
from tests import esdf_fe_check as fc
from tests import test_esdf_reference_gpu as te
from tests.test_esdf_options_gpu import _freespace_scan
from tests.golden import reference_pins as pins

pytestmark = pytest.mark.gpu


# ------------------------------------------------------------------ synthetic layers
SYN_KEYS = ([f"{s}/{v}" for s in ("point", "point_inside") for v in (16, 4, 1)]
            + [f"{s}/{v}" for s in ("two_points", "plane", "tilted") for v in (16, 4)] + ["hairpin/4"])


def _device_synthetic(g, d, vps, ekw, voxel=fc.SYN_VOXEL):
    """The device layers of a synthetic TSDF layer: (TSDF layer, ESDF layer, EsdfIntegrator)."""
    idx, vox = fc.tsdf_blocks(g, d, vps)
    tsdf = vb.Layer(voxel, vps)
    vb.TsdfIntegratorFactory.create("merged", vb.TsdfIntegratorConfig(default_truncation_distance=fc.SYN_FREE), tsdf)
    esdf = vb.Layer(voxel, vps, voxel_type="esdf")
    eint = vb.EsdfIntegrator(vb.EsdfIntegratorConfig(**ekw), tsdf, esdf)
    tsdf.insertBlocks(idx, vox.view(vb.TSDF_DTYPE))
    return tsdf, esdf, eint


def synthetic_reference_side(key, lib):
    scene, vps = key.split("/")
    g, d = fc.synthetic(scene)
    omap = fc.oracle_layer(lib, g, d, int(vps), fc.SYN_EKW)
    return omap.blocks(1), pins.map_digest(omap, (po.LAYER_TSDF, po.LAYER_ESDF))


def _layer_bytes(blocks):
    return b"".join(np.array(k, np.int32).tobytes() + blocks[k].tobytes() for k in sorted(blocks))


@pytest.mark.parametrize("key", SYN_KEYS)
def test_synthetic(key):
    scene, vps = key.split("/")
    vps = int(vps)
    ref, digest = synthetic_reference_side(key, pins.lib())
    pins.check(f"esdf_fe/synthetic/{key}", digest)
    g, d = fc.synthetic(scene)
    _, esdf, eint = _device_synthetic(g, d, vps, fc.SYN_EKW)
    eint.updateFromTsdfLayerBatch()
    dev = esdf.blocks()
    out = {}
    for side, blocks in (("device", dev), ("reference", ref)):
        rep = fc.counts(fc.fe_check(blocks, fc.SYN_VOXEL, vps, fc.SYN_EKW))
        e = fc.euclidean(blocks, fc.SYN_VOXEL, vps, fc.SYN_EKW)
        out[side] = (rep, e)
        print(key, side, rep, {k: v for k, v in e.items() if k not in ("edt", "grid", "under")})
    assert sorted(dev) == sorted(ref)
    for side, (rep, e) in out.items():
        assert rep["a"] == 0 and rep["range"] == 0, (side, rep)
        assert rep["r_fixed_other"] == rep["r_seeded"] == rep["r_unit"] == rep["r_other"] == 0, (side, rep)
        assert rep["t"] == 0 and len(e["under"]) == 0, (side, rep)
    rep, e = out["device"]
    if scene in ("point", "point_inside", "two_points", "hairpin", "plane"):
        # one fixed voxel, two, a plane one voxel thick on each side, or a path: the vector propagation is exact
        assert e["exact"] == e["compared"] == rep["reached"], (rep, e)
    if scene in ("point", "point_inside"):
        assert rep["reached"] == len(g) - 1
    if scene == "tilted":
        # measured on one H100: device and reference both 3 of 3505 voxels off the EDT, by at most 1.5 mm
        assert e["over_tol"] <= out["reference"][1]["over_tol"] + 3, (e, out["reference"][1])
        assert e["max"] <= out["reference"][1]["max"] + 0.01
    if scene == "hairpin":
        # the way back: every candidate from the turn has a negative step (cc:423-425), so it stays unreached
        grid = e["grid"]
        back = grid.lookup(np.array([(x, 3, 0) for x in range(fc.HAIRPIN_L)], np.int64))
        assert (back >= 0).all() and (grid.d[back] == np.float32(fc.SYN_EKW["default_distance_m"])).all()
        assert _layer_bytes(dev) == _layer_bytes(ref)


# the parent code's range: a line of 2 x 2 voxels along x in a 1 x 1 x N strip of blocks, fixed at one end
RANGE_CASES = {"minus_512": (-1, 512, True), "minus_513": (-1, 513, False),
               "plus_511": (1, 511, True), "plus_512": (1, 512, False)}
RANGE_VOXEL, RANGE_VPS = 0.1, 16


def _strip(direction, length):
    """Voxels x = 0..length (y, z in {0, 1}) with the fixed voxels at x = 0 (direction -1: chains run to +x and their
    parents to -length) or at x = length (direction +1: parents up to +length)."""
    x = np.arange(length + 1)
    g = np.stack(np.meshgrid(x, np.arange(2), np.arange(2), indexing="ij"), -1).reshape(-1, 3).astype(np.int64)
    fixed_x = 0 if direction < 0 else length
    d = np.where(g[:, 0] == fixed_x, np.float32(0.01), np.float32(fc.SYN_FREE)).astype(np.float32)
    mx = float(np.float32(RANGE_VOXEL * (length + 8)))
    return g, d, dict(fc.SYN_EKW, max_distance_m=mx, default_distance_m=mx)


@pytest.mark.parametrize("case", list(RANGE_CASES))
def test_parent_range(case):
    """A chain whose parent reaches -512 succeeds and passes the checks; one that reaches +512 (or -513) fails the
    update with VBX_E_CAPACITY: the parent code holds [-512, 511]."""
    direction, length, ok = RANGE_CASES[case]
    g, d, ekw = _strip(direction, length)
    _, esdf, eint = _device_synthetic(g, d, RANGE_VPS, ekw, RANGE_VOXEL)
    if not ok:
        with pytest.raises(vb.VoxbloxError, match=r"parent vector component left \[-512, 511\]"):
            eint.updateFromTsdfLayerBatch()
        return
    eint.updateFromTsdfLayerBatch()
    blocks = esdf.blocks()
    rep = fc.fe_check(blocks, RANGE_VOXEL, RANGE_VPS, ekw)
    print(case, fc.counts(rep))
    assert len(rep["a"]) == 0 and len(rep["range"]) == 0 and len(rep["t"]) == 0, fc.counts(rep)
    assert rep["reached"] == len(g) - 4 and len(rep["r_fixed_same"]) == rep["reached"], fc.counts(rep)
    grid = fc.Grid(blocks, RANGE_VPS)
    assert grid.parent[:, 0].min() == (-length if direction < 0 else 0)
    assert grid.parent[:, 0].max() == (0 if direction < 0 else length)


# ------------------------------------------------------------------ room and cylinder scenes
# scene -> (voxel size, truncation, voxels per side, max_distance_m, scans); (e) runs where it is affordable
SCENES = {
    "room_small": (0.1, 0.4, 16, 2.0, te.ROOM_SMALL["scans"]),
    "room_small_vps8": (0.1, 0.4, 8, 2.0, te.ROOM_SMALL["scans"]),
    "room_small_vps4": (0.1, 0.4, 4, 2.0, te.ROOM_SMALL["scans"]),
    "room_full_640x480": (0.05, 0.2, 16, 2.0, te.ROOM_FULL["scans"]),
    "cylinder_0.2": (0.2, 0.8, 16, 4.0, te._gt_scans),
    "cylinder_0.1": (0.1, 0.4, 16, 4.0, te._gt_scans),
}
CONFIGS = {"min_diff_zero": dict(min_diff_m=0.0, multi_queue=1), "ros_default": dict(min_diff_m=1e-3, multi_queue=0)}
# incremental: the update after which setFullEuclidean(true) is called (0: on from the start), as in
# test_esdf_options_gpu.FE_SWITCH_AFTER
SWITCH_AFTER = {"room_small": 1, "room_small_vps8": 1, "room_small_vps4": 1, "room_full_640x480": 0}
KEYS = ([f"batch/{c}/{s}" for c in CONFIGS for s in SCENES]
        + [f"incremental/{c}/{s}" for c in CONFIGS for s in SWITCH_AFTER]
        + [f"raise/{c}/room_small" for c in CONFIGS])
PIN_KEYS = [f"synthetic/{k}" for k in SYN_KEYS] + KEYS


def _case(key):
    kind, config, scene = key.split("/")
    voxel, trunc, vps, max_d, scans = SCENES[scene]
    switch = SWITCH_AFTER.get(scene, 0) if kind == "incremental" else 0
    ekw = dict(max_distance_m=max_d, default_distance_m=max_d, min_distance_m=trunc / 2,
               full_euclidean_distance=int(switch == 0), **CONFIGS[config])
    return kind, voxel, trunc, vps, ekw, scans, switch


def _drive(key, scans, integrate, update, set_fe, esdf_blocks):
    """One case on either side.  Returns the checked (full-Euclidean) updates as (incremental, before, after)."""
    kind, _, _, _, _, _, switch = _case(key)
    out = []

    def checked(fn, incremental):
        before = esdf_blocks()
        fn()
        out.append((incremental, before, esdf_blocks()))

    if kind == "batch":
        for s in scans:
            integrate(s, False)
        checked(lambda: update(True), False)
    elif kind == "incremental":
        for k, s in enumerate(scans):
            integrate(s, False)
            if k >= switch:
                checked(lambda: update(False), True)
            else:
                update(False)
            if k + 1 == switch:
                set_fe()
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
    kind, voxel, trunc, vps, ekw, scans, _ = _case(key)
    omap = po.OracleMap(lib, po.TsdfConfig(default_truncation_distance=trunc, integrator_threads=1), voxel, vps)
    omap.esdf_create(po.EsdfConfig(**ekw))
    steps = _drive(key, scans(), lambda s, free: omap.integrate(2, s, freespace=free),
                   lambda batch: omap.esdf_update(batch=batch, clear_updated_flag=True),
                   lambda: omap.esdf_set_full_euclidean(True), lambda: omap.blocks(1))
    h = pins.map_digest(omap, (po.LAYER_TSDF,))
    for _, _, after in steps:
        for i in sorted(after):
            h += pins.array_digest(np.array(i, np.int32), after[i])
    return steps, pins.array_digest(np.frombuffer(h.encode(), np.uint8))


def device_side(key):
    kind, voxel, trunc, vps, ekw, scans, _ = _case(key)
    tsdf = vb.Layer(voxel, vps)
    integ = vb.TsdfIntegratorFactory.create(
        "merged", vb.TsdfIntegratorConfig(default_truncation_distance=trunc, integrator_threads=1), tsdf)
    esdf = vb.Layer(voxel, vps, voxel_type="esdf")
    eint = vb.EsdfIntegrator(vb.EsdfIntegratorConfig(**ekw), tsdf, esdf)
    return _drive(key, scans(), lambda s, free: integ.integratePointCloud((s[2], s[3]), s[0], s[1], freespace_points=free),
                  lambda batch: eint.updateFromTsdfLayerBatch() if batch else eint.updateFromTsdfLayer(True),
                  lambda: eint.setFullEuclidean(True), esdf.blocks)


def _reports(steps, key):
    kind, voxel, _, vps, ekw, _, _ = _case(key)
    reps = []
    for incremental, before, after in steps:
        rep = fc.counts(fc.fe_check(after, voxel, vps, ekw, incremental=incremental,
                                    before=before if incremental else None))
        if not incremental:
            e = fc.euclidean(after, voxel, vps, ekw, max_pairs=2e9)
            if e is not None:
                rep.update({f"edt_{k}": (len(v) if k == "under" else v) for k, v in e.items() if k not in ("edt", "grid")})
        reps.append(rep)
    return reps


@pytest.mark.parametrize("key", KEYS)
def test_fe_scene(key):
    kind = key.split("/")[0]
    ref_steps, digest = reference_side(key, pins.lib())
    pins.check(f"esdf_fe/{key}", digest)
    dev, ref = _reports(device_side(key), key), _reports(ref_steps, key)
    for k, (d, r) in enumerate(zip(dev, ref)):
        print(key, "update", k, "\n  device   ", d, "\n  reference", r)
    assert len(dev) == len(ref)
    voxel = SCENES[key.split("/")[2]][0]
    if kind == "batch":
        for d, r in zip(dev, ref):
            assert d["a"] == 0 and d["range"] == 0, d
            # every chain starts at a fixed voxel (of either sign: the mixed rule keeps the root across the surface)
            assert d["r_seeded"] == d["r_unit"] == d["r_other"] == 0, d
            # (t) breaks only where a chain crossed the surface twice through the mixed rule, which restarts the value
            # but not the root; measured on one H100: 0 on both sides on cylinder_0.2, elsewhere the device at most
            # 1.47x the reference's count (room_full_640x480, ROS defaults: 9805 vs 6692)
            if key.endswith("cylinder_0.2"):
                assert d["t"] == 0 == r["t"], (d, r)
            assert d["t"] <= 2 * r["t"], (d, r)
            if "edt_compared" in d:
                # below the EDT only off the telescoping identity
                assert d["edt_under"] <= d["t"], d
                # measured: the device's p99 of |d| - EDT at most 0.011 voxel above the reference's, its max at most
                # 0.08 voxel above
                assert d["edt_p99"] <= r["edt_p99"] + 0.1 * voxel, (d, r)
                assert d["edt_max"] <= r["edt_max"] + 0.25 * voxel, (d, r)
    else:
        total = {c: (sum(d[c] for d in dev), sum(r[c] for r in ref))
                 for c in fc.A_CLASSES + fc.ROOT_CLASSES + fc.STALE_CLASSES + ("range", "t")}
        print(key, "classes (device, reference):", total)
        for d in dev:
            assert d["a_other"] == 0 and d["range"] == 0, d
        assert total["a_mixed"][0] <= total["a_mixed"][1], total
        # unchanged voxels whose rounded parent direction points at a voxel whose |d| rose: the raise test of
        # cc:339-347 resets those, but a reset voxel can take its old word back from a chain the test did not reach.
        # Measured on one H100: the device 46-235 per case, the reference 164-720; at most 1.17x the reference's
        # (raise, min_diff 0: 235 vs 201)
        assert total["s_parent_raised"][0] <= 1.5 * total["s_parent_raised"][1] + 50, total
