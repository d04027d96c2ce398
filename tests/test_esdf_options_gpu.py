"""-m gpu: the EsdfIntegrator::Config options the other ESDF tests leave at their defaults -- full_euclidean_distance,
add_occupied_crust and a min_weight above many voxels' TSDF weight -- on the device against the REFERENCE's own
EsdfIntegrator (oracle/_ref), where that library exists, else the restatement held to its recorded digests
(tests/golden/reference_pins.py).

Full-Euclidean mode propagates voxel_size * (|parent - dir| - |parent|) from a voxel's parent vector
(esdf_integrator.cc:414-426), so the reference's own result depends on its pop order, and no parallel order
reproduces it.  Two kinds of check remain:
 * flags and block sets are order free: exact;
 * the parent vector is a chain of sums, so it points from a voxel to the voxel its chain started from
   (root = v + parent(v)), and along a same-sign chain the steps telescope:
       distance(v) == distance(root) + sign(distance(v)) * voxel_size * |parent(v)|
   for every voxel whose root is a fixed voxel of its own sign, in any visiting order.  A voxel whose distance
   and parent came from two different sources breaks it.  Mixed-sign assignments (cc:458-488) and incremental
   updates (roots that are seeded or earlier-lowered voxels) restart chains, so it is asserted on batch updates
   of the ground-truth scenes; elsewhere the distances get statistical bounds.
The bounds are measured values plus a margin; every test prints the measured numbers."""
import functools

import numpy as np
import pytest

from oracle import pyoracle as po
from tests import test_esdf_reference_gpu as te
from tests.golden import reference_pins as pins

pytestmark = pytest.mark.gpu


def _room_ekw(scene, **kw):
    """The reference test's ESDF configuration (min_diff 0, multi_queue) on a room scene."""
    return dict(max_distance_m=2.0, default_distance_m=2.0, min_distance_m=te.SCENES[scene]["trunc"] / 2,
                min_diff_m=0.0, multi_queue=1, **kw)


# incremental full-Euclidean sequences: the update after which setFullEuclidean(True) is called (0: on from the start)
FE_SWITCH_AFTER = {"room_small": 1, "room_full_640x480": 0}
CRUST_SPLIT = 2         # crust: batch update after this many scans, incremental update after the rest
MIN_WEIGHT_QUANTILE = 0.3


def _freespace_scan(scan, stretch=1.5):
    """`scan` with every ray stretched past its surface; integrated with freespace_points, it re-observes the
    old surface as free space (what a moved object leaves behind), so fixed voxels turn free and are raised."""
    pts, cols, q, t = scan
    return (pts * np.float32(stretch)).astype(np.float32), cols, q, t


def _scans(key):
    what, scene = key.split("/")
    scans = te.SCENES[scene]["scans"]()
    if what == "fe_raise":
        return scans, [_freespace_scan(scans[-1])] * 2
    return scans, []


def _min_weight(tsdf_weights):
    """A min_weight that a MIN_WEIGHT_QUANTILE share of the observed TSDF voxels fall below."""
    w = tsdf_weights[tsdf_weights > 0]
    return float(np.quantile(w, MIN_WEIGHT_QUANTILE))


def _tsdf_weights(omap):
    return np.concatenate([omap.block(i)[0]["weight"] for i in omap.block_indices()])


def _run(esdf_update, integrate, key, scans, free):
    """Drives one case through either side: `integrate(scan, freespace)`, `esdf_update(batch)`, and
    `esdf_update("fe")` for setFullEuclidean(True)."""
    what, scene = key.split("/")
    if what == "fe_batch":
        for s in scans:
            integrate(s, False)
        esdf_update(True)
    elif what in ("fe_incremental", "fe_raise"):
        switch = FE_SWITCH_AFTER[scene] if what == "fe_incremental" else 0
        if switch == 0:
            esdf_update("fe")
        for k, s in enumerate(list(scans) + list(free)):
            integrate(s, k >= len(scans))
            esdf_update(False)
            if k + 1 == switch:
                esdf_update("fe")
    elif what == "crust_batch":
        for s in scans[:CRUST_SPLIT]:
            integrate(s, False)
        esdf_update(True)
    elif what == "crust":
        for s in scans[:CRUST_SPLIT]:
            integrate(s, False)
        esdf_update(True)
        for s in scans[CRUST_SPLIT:]:
            integrate(s, False)
        esdf_update(False)
    elif what in ("min_weight_incremental", "min_weight_batch"):
        for s in scans:
            integrate(s, False)
            if what == "min_weight_incremental":
                esdf_update(False)
        if what == "min_weight_batch":
            esdf_update(True)
    else:
        raise KeyError(key)


def _ekw(key, min_weight=None):
    what, scene = key.split("/")
    if what.startswith("fe_"):
        return _room_ekw(scene, full_euclidean_distance=int(what == "fe_batch"))
    if what.startswith("crust"):
        return _room_ekw(scene, add_occupied_crust=1)
    return _room_ekw(scene, min_weight=min_weight)


def _oracle_side(lib, key, scans, free, ekw):
    sc = te.SCENES[key.split("/")[1]]
    omap = po.OracleMap(lib, po.TsdfConfig(default_truncation_distance=sc["trunc"], integrator_threads=1), sc["voxel"], 16)
    omap.esdf_create(po.EsdfConfig(**ekw))

    def esdf_update(batch):
        if batch == "fe":
            omap.esdf_set_full_euclidean(True)
        else:
            omap.esdf_update(batch=batch, clear_updated_flag=True)

    _run(esdf_update, lambda s, free_: omap.integrate(2, s, freespace=free_), key, scans, free)
    return omap


def reference_side(key, lib):
    """The oracle side of case `key` ("<case>/<scene>"): the scans, the oracle map and the digest of its TSDF and
    ESDF layers.  min_weight cases pick their threshold from the TSDF map of the same scans (it goes into the
    digest too)."""
    scans, free = _scans(key)
    min_weight = None
    if key.startswith("min_weight"):
        sc = te.SCENES[key.split("/")[1]]
        tmap = po.OracleMap(lib, po.TsdfConfig(default_truncation_distance=sc["trunc"], integrator_threads=1),
                            sc["voxel"], 16)
        for s in scans:
            tmap.integrate(2, s)
        min_weight = _min_weight(_tsdf_weights(tmap))
    omap = _oracle_side(lib, key, scans, free, _ekw(key, min_weight))
    h = pins.map_digest(omap, (po.LAYER_TSDF, po.LAYER_ESDF)) + repr(min_weight)
    return (scans, free, min_weight), omap, pins.array_digest(np.frombuffer(h.encode(), np.uint8))


PIN_KEYS = ([f"fe_incremental/{sc}" for sc in te.SCENES] + [f"fe_batch/{sc}" for sc in te.SCENES]
            + ["fe_raise/room_small", "crust_batch/room_small", "crust/room_small",
               "min_weight_incremental/room_small", "min_weight_batch/room_small"])


def _case(key):
    """(device ESDF layer, device TSDF layer, EsdfIntegrator, oracle map, min_weight, counters of the last update)."""
    (scans, free, min_weight), omap, digest = reference_side(key, pins.lib())
    pins.check(f"esdf_options/{key}", digest)
    sc = te.SCENES[key.split("/")[1]]
    tsdf, integ, esdf, eint = te._device(sc["voxel"], sc["trunc"], _ekw(key, min_weight))
    last = {}

    def esdf_update(batch):
        if batch == "fe":
            eint.setFullEuclidean(True)
            return
        if batch:
            eint.updateFromTsdfLayerBatch()
        else:
            eint.updateFromTsdfLayer(True)
        last.update(eint.counters())

    def integrate(s, free_):
        integ.integratePointCloud((s[2], s[3]), s[0], s[1], freespace_points=free_)

    _run(esdf_update, integrate, key, scans, free)
    return esdf, tsdf, eint, omap, min_weight, last


def _voxels(esdf, omap):
    """Both ESDF layers' voxels, every block (the block sets must be equal)."""
    gi, oi = esdf.getAllAllocatedBlocks(), omap.block_indices(1)
    assert gi.shape == oi.shape and (gi == oi).all()
    gv, _ = esdf.getBlocks(gi)
    return gv, np.stack([omap.block(i, 1)[0] for i in oi])


def _assert_flags_exact(gv, ov):
    for flag in ("observed", "hallucinated", "fixed"):
        assert (gv[flag] == ov[flag]).all(), flag


def _fe_room_stats(esdf, omap, voxel):
    """_diff_stats, plus the sign agreement over the voxels the reference holds at a non-zero distance."""
    st = te._diff_stats(esdf, omap, voxel, 0.0)
    gv, ov = _voxels(esdf, omap)
    obs = ov["observed"] != 0
    dg, do = gv["distance"][obs], ov["distance"][obs]
    nz = do != 0
    st["reference_zeros"] = int((~nz).sum())
    st["sign_equal_nonzero"] = float((np.sign(dg[nz]) == np.sign(do[nz])).mean())
    return st


def _assert_fe_room_bounds(st, voxel):
    """Full Euclidean on the room scenes.  A step from a voxel's parent can be 0 (|parent - dir| == |parent|), and
    where that step meets a voxel of the other sign the reference assigns signum(distance) * 0 (cc:475-486): the
    free voxel becomes 0.0, counts as inside from then on (cc:444) and takes inside values from its neighbours.
    The device keeps only candidates of the voxel's own sign, so those voxels and what propagates from them differ
    (measured: the reference holds 455 non-fixed exact zeros of 7897 observed voxels in room_small, 928 of 46708 in
    room_full_640x480; sign agreement 0.918-0.98, within one voxel 0.50-0.76, rmse 1.2-2.7 voxels, max 1.37 m)."""
    assert st["sign_equal_nonzero"] >= 0.99, st
    assert st["sign_equal"] >= 0.9, st
    assert st["within_one_voxel"] >= 0.45, st
    assert st["rmse_m"] <= 3.5 * voxel, st
    assert st["max_abs_err_m"] < 2.0, st


def _assert_room_bounds(st, voxel):
    """The bounds of the room tests in test_esdf_reference_gpu.py."""
    assert st["sign_equal"] == 1.0, st
    assert st["within_one_voxel"] >= 0.995, st
    assert st["rmse_m"] <= 0.3 * voxel, st
    assert st["max_abs_err_m"] < 2.0, st


# ------------------------------------------------------------------ parent-root identity
def parent_root_check(blocks, voxel, max_distance, vps=16):
    """The telescoping identity above, in float64, on one ESDF layer ({block index: voxels}).  Candidates are the
    voxels that are observed, not fixed, inside +-max_distance and have a non-zero parent; `rooted` those whose
    root (v + parent) is an observed fixed voxel of the same sign; `violations` the rooted voxels off the identity
    by more than 1e-5 * max(1, |parent|) m."""
    idx = np.array(list(blocks), np.int64).reshape(-1, 3)
    vox = np.stack(list(blocks.values())).reshape(-1)
    lin = np.arange(vps ** 3)
    local = np.stack([lin % vps, (lin // vps) % vps, lin // (vps * vps)], 1)
    g = (idx[:, None, :] * vps + local[None]).reshape(-1, 3)

    def key(c):
        c = c + (1 << 26)
        return (c[:, 0] << 54) | (c[:, 1] << 27) | c[:, 2]

    keys = key(g)
    order = np.argsort(keys)
    d = vox["distance"].astype(np.float64)
    obs, fixed, par = vox["observed"] != 0, vox["fixed"] != 0, vox["parent"].astype(np.int64)
    cand = obs & ~fixed & (np.abs(d) < max_distance) & (par != 0).any(1)
    ci = np.nonzero(cand)[0]
    rk = key(g[ci] + par[ci])
    pos = np.minimum(np.searchsorted(keys, rk, sorter=order), len(keys) - 1)
    ri = order[pos]
    found = keys[ri] == rk
    rooted = found & obs[ri] & fixed[ri] & ((d[ri] > 0) == (d[ci] > 0))
    vi, ri = ci[rooted], ri[rooted]
    plen = np.sqrt((par[vi] ** 2).sum(1).astype(np.float64))
    pred = d[ri] + np.where(d[vi] > 0, 1.0, -1.0) * voxel * plen
    err = np.abs(d[vi] - pred)
    bad = err > 1e-5 * np.maximum(1.0, plen)
    return {"candidates": int(ci.size), "rooted": int(vi.size), "rooted_fraction": float(vi.size / max(1, ci.size)),
            "violations": int(bad.sum()), "max_err_m": float(err.max()) if err.size else 0.0,
            "max_parent_len": float(plen.max()) if plen.size else 0.0}


@functools.lru_cache(maxsize=None)
def _gt_case(voxel):
    """The ground-truth scene of test_esdf_reference_gpu.py, full-Euclidean batch: (device layer blocks, reference
    maps: quasi-Euclidean incremental, batch, full-Euclidean batch)."""
    scans, maps, digest = te.reference_side(f"ground_truth/{voxel}", pins.lib())
    pins.check(f"esdf/ground_truth/{voxel}", digest)
    return te.gt_batch_layer(scans, voxel, True).blocks(), maps


@pytest.mark.parametrize("voxel", te.GT_VOXELS)
def test_full_euclidean_ground_truth(voxel):
    """The third layer of SdfIntegratorsTest.EsdfIntegrators (test_sdf_integrators.cc:193-272): a full-Euclidean
    batch update of the cylinder-on-plane scene against the analytic distance field, beside the reference's."""
    max_d = te._gt_config(voxel)[1]["max_distance_m"]
    blocks, (ref_inc, _, ref_fe) = _gt_case(voxel)
    fe = te._gt_errors(blocks, voxel, max_d)
    r_fe = te._gt_errors(ref_fe.blocks(1), voxel, max_d)
    r_inc = te._gt_errors(ref_inc.blocks(1), voxel, max_d)
    print("voxel", voxel, "device full-Euclidean batch", fe, "| reference", r_fe, "| reference incremental", r_inc)
    assert fe["min_error"] <= 1e-4
    assert fe["max_error"] < max_d
    assert fe["rmse"] < max_d * voxel
    assert fe["voxels"] == r_inc["voxels"] == r_fe["voxels"]
    assert fe["rmse"] <= r_fe["rmse"] * 1.02 + 1e-4


@pytest.mark.parametrize("voxel", te.GT_VOXELS)
def test_full_euclidean_parent_root_identity(voxel):
    """Every device voxel with a same-sign fixed root satisfies the telescoping identity where every such voxel of
    the reference does (0.2 m); where the reference has exceptions, the device has no larger a share of them plus
    0.5 percentage points.  The share of voxels that have such a root is the reference's within 2 percentage
    points.  The check is run on the reference's map first."""
    max_d = te._gt_config(voxel)[1]["max_distance_m"]
    blocks, (_, _, ref_fe) = _gt_case(voxel)
    ref = parent_root_check(ref_fe.blocks(1), voxel, max_d)
    dev = parent_root_check(blocks, voxel, max_d)
    print("voxel", voxel, "parent-root identity: device", dev, "| reference", ref)
    assert ref["rooted"] > 0
    if ref["violations"] == 0:
        assert dev["violations"] == 0, dev
    else:
        # at 0.1 m some chains of the reference itself cross the surface twice (mixed-sign assignments) and come
        # back to a root of their own sign: 8751 of its 278677 rooted voxels (3.1 %)
        assert dev["violations"] <= (ref["violations"] / ref["rooted"] + 0.005) * dev["rooted"], (dev, ref)
    assert dev["rooted_fraction"] >= ref["rooted_fraction"] - 0.02, (dev, ref)


@pytest.mark.parametrize("scene", list(te.SCENES))
@pytest.mark.parametrize("mode", ["fe_incremental", "fe_batch"])
def test_full_euclidean_room(mode, scene):
    """Full-Euclidean updates of the room scenes: incremental after every scan (room_small switches
    setFullEuclidean(True) on after its first update) and batch."""
    sc = te.SCENES[scene]
    esdf, _, _, omap, _, last = _case(f"{mode}/{scene}")
    gv, ov = _voxels(esdf, omap)
    _assert_flags_exact(gv, ov)
    st = _fe_room_stats(esdf, omap, sc["voxel"])
    print(mode, scene, st, "counters", last)
    _assert_fe_room_bounds(st, sc["voxel"])


def test_full_euclidean_raise():
    """Full-Euclidean incremental updates of room_small, then two scans whose rays run past the old surface,
    integrated as free space: the surface's fixed voxels turn free and raise their descendants (cc:305-369, with
    the full-Euclidean parent test of cc:339-347)."""
    sc = te.SCENES["room_small"]
    esdf, _, _, omap, _, last = _case("fe_raise/room_small")
    gv, ov = _voxels(esdf, omap)
    _assert_flags_exact(gv, ov)
    st = _fe_room_stats(esdf, omap, sc["voxel"])
    print("fe_raise room_small", st, "counters", last)
    assert last["raise"] > 0 and last["raised_voxels"] > 0, last
    _assert_fe_room_bounds(st, sc["voxel"])


@pytest.mark.parametrize("stage", ["crust_batch", "crust"])
def test_add_occupied_crust(stage):
    """add_occupied_crust: a batch update marks every unobserved voxel of every TSDF block observed, hallucinated
    and at -default_distance (cc:153-164); an incremental update after more scans then re-classifies the crust the
    new scans observe.  Flags are exact on every voxel; crust voxels no propagation reached hold exactly
    -default_distance_m."""
    sc = te.SCENES["room_small"]
    ekw = _room_ekw("room_small")
    esdf, _, _, omap, _, last = _case(f"{stage}/room_small")
    gv, ov = _voxels(esdf, omap)
    _assert_flags_exact(gv, ov)
    crust = ov["hallucinated"] != 0
    default = np.float32(-ekw["default_distance_m"])
    unreached_ref, unreached_dev = crust & (ov["distance"] == default), crust & (gv["distance"] == default)
    st = te._diff_stats(esdf, omap, sc["voxel"], 0.0)
    print(stage, st, "crust voxels", int(crust.sum()), "unreached: reference", int(unreached_ref.sum()),
          "device", int(unreached_dev.sum()), "counters", last)
    assert crust.sum() > 0
    assert (gv["distance"][crust] <= 0).all() and (gv["distance"][crust] >= default).all()
    # which crust voxels a propagation reaches depends on the sign-conflict voxels next to them (order dependent
    # in the reference, see test_esdf_reference_gpu.py); measured: 11 of 1583 (batch) and 6 of 1291 differ
    assert (unreached_dev != unreached_ref).sum() <= 0.02 * unreached_ref.sum()
    _assert_room_bounds(st, sc["voxel"])


@pytest.mark.parametrize("mode", ["min_weight_incremental", "min_weight_batch"])
def test_min_weight_leaves_light_voxels_alone(mode):
    """min_weight above the TSDF weight of a MIN_WEIGHT_QUANTILE share of the observed voxels: those voxels are
    unobserved for the ESDF (cc:153-164) and keep the ESDF voxel they had, bit for bit."""
    sc = te.SCENES["room_small"]
    esdf, tsdf, _, omap, min_weight, last = _case(f"{mode}/room_small")
    gv, ov = _voxels(esdf, omap)
    _assert_flags_exact(gv, ov)
    assert (tsdf.getAllAllocatedBlocks() == esdf.getAllAllocatedBlocks()).all()
    tw, _ = tsdf.getBlocks(esdf.getAllAllocatedBlocks())
    light = (tw["weight"] > 0) & (tw["weight"] < min_weight)
    share = float(light.sum() / max(1, (tw["weight"] > 0).sum()))
    st = te._diff_stats(esdf, omap, sc["voxel"], 0.0)
    print(mode, "min_weight", min_weight, "light share", share, st, "counters", last)
    assert share >= 0.2
    assert gv[light].tobytes() == ov[light].tobytes()
    assert (gv["observed"][light] == 0).all()
    _assert_room_bounds(st, sc["voxel"])
