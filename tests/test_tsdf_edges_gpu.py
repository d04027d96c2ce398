"""-m gpu: Simple and Merged end to end, bit for bit against the REFERENCE's own integrators (oracle/_ref,
one integrator thread) where that library exists, else the restatement held to the reference's recorded
digests (tests/golden/reference_pins.py), on what the other parity tests never reach:

 * a prior map: blocks whose voxels sit at the states a map loaded from a file, pushed through setLayer or
   saved under another max_weight or truncation can hold -- integer weights just below 2^24 and 2^22,
   (T, max_weight), (T, 2 max_weight), 3T, a weight below 1e-6, -0.0 -- inserted on the device and
   deserialised on the oracle, then integrated into;
 * camera-frame depths at the weight function's edges (z = 0, 5e-7 and 2e-6, points 400x farther away) with
   non-constant weights and min_ray_length_m = 0: zero weights, weights below kEpsilon that the Merged fold
   skips, weights near 1e11, big bundles whose weights are all 0 or all near 1e11, a big bundle that the
   Merged fold must fold again with IEEE division, and points within 0.1 m of the sensor;
 * the bundles whose mean the Merged fold folds again with IEEE division, in each shape that walk meets: fewer
   than 32 members, the first live member past the first chunk, live and weight-0 members alternating, and a
   clearing bundle;
 * a truncation distance at or below the voxel size (the weight drop-off's denominator is 0 or negative);
 * max_weight of 1e-7 (a voxel can never rest), 1 and 1e30."""
import numpy as np
import pytest

import voxblox_b200 as vb
from oracle import pyoracle as po
from tests.golden import reference_pins as pins
from tests.parity import compare_tsdf
from voxblox_b200 import scenes

pytestmark = pytest.mark.gpu

ROOM_T, ROOM_VS = 0.4, 0.1


def _room(n=3):
    return scenes.c3_room_sequence(n_scans=n, width=96, height=72)


def _lidar_extreme_z():
    s = scenes.c5_lidar_scan(0)
    pts = s[0][::8].copy()
    pts[::50, 2] = 0.0           # weight 0
    pts[1::50, 2] = 5e-7         # |z| <= kEpsilon: weight 0
    pts[2::50, 2] = 2e-6         # weight ~2.5e11
    pts[3::97] *= 400.0          # far away: weights below 1e-6 once |z| > 1000
    # dense clusters, each inside one voxel, so each is one big Merged bundle (>= 256 members):
    rng = np.random.default_rng(11)
    jitter = lambda n, k: rng.uniform(0.0, 1e-4, (n, k)).astype(np.float32)
    F = np.float32
    clusters = [
        # z = 0: every weight 0, the fold skips every member
        np.c_[F(0.55) + jitter(400, 2), np.zeros(400, F)],
        # z ~ 2e-6: weights ~2.5e11
        np.c_[F(0.55) + jitter(400, 2), rng.uniform(1.5e-6, 2.5e-6, 400).astype(F)],
        # camera-frame x exactly 0: the running mean of x has a zero dividend, which the fold's three-operation
        # division does not trust, so the bundle is folded again with IEEE division (refolded_bundles)
        np.c_[np.zeros(600, F), F(0.55) + jitter(600, 1), F(1.5) + jitter(600, 1)],
        # about 6 cm from the sensor: valid with min_ray_length_m = 0 only
        np.c_[F(0.03) + jitter(300, 2), F(0.04) + jitter(300, 1)],
    ]
    extra = np.concatenate(clusters).astype(F)
    pts = np.concatenate([pts, extra])
    cols = np.concatenate([s[1][::8], rng.integers(0, 256, (len(extra), 4)).astype(np.uint8)])
    return [(pts, cols, s[2], s[3])]


def _refold_cluster(shape):
    """One scan of one dense cluster with camera-frame x = 0 (so the Merged fold folds its mean again with IEEE
    division), inside one voxel under C1's pose, shaped for what that refold walks: under 1024 points, so that list
    order is array order, and weights of 0 at camera-frame z = 0 next to live ones at z ~ 5 mm."""
    rng = np.random.default_rng(17)
    F = np.float32
    jitter = lambda n: rng.uniform(0.0, 1e-4, n).astype(F)
    live_z = lambda n: F(0.005) + jitter(n)
    if shape == "short":          # fewer than 32 members: one partial chunk
        z = F(1.55) + jitter(20)
    elif shape == "late_live":    # the first live member is past the first chunk
        z = np.r_[np.zeros(45, F), live_z(60)]
    elif shape == "alternating":  # live and weight-0 members alternate: partial live masks in every chunk
        z = np.where(np.arange(100) % 2 == 0, F(0), live_z(100)).astype(F)
    else:                         # "clearing": beyond max_ray_length_m, so only the first member is taken
        z = F(6.05) + jitter(50)
    n = len(z)
    pts = np.c_[np.zeros(n, F), F(0.55) + jitter(n), z].astype(F)
    cols = rng.integers(0, 256, (n, 4)).astype(np.uint8)
    _, _, q, t = scenes.c1_planar_wall()
    return [(pts, cols, q, t)]


def _mutate_prior(words, T, max_weight, seed):
    """Voxels of a serialised block (3 words each) set to the edge states, one in eight of each kind."""
    w = words.reshape(-1, 3).copy()
    d = w[:, 0].view(np.float32)
    wt = w[:, 1].view(np.float32)
    obs = wt > 0
    pick = np.random.default_rng(seed).integers(0, 8, size=len(d))
    F = np.float32
    wt[(pick == 0) & obs] = F(16777213.0)
    wt[(pick == 1) & obs] = F(4194303.0)
    sel = (pick == 2) & obs
    d[sel], wt[sel] = F(T), F(max_weight)
    sel = (pick == 3) & obs
    d[sel], wt[sel] = F(T), F(max_weight) * F(2)
    d[(pick == 4) & obs] = F(3 * T)
    wt[(pick == 5) & obs] = F(5e-7)
    d[(pick == 6) & obs] = F(-0.0)
    return w.reshape(-1)


# key -> voxel size, config, scans, whether a prior map is built from the first scan, what the counters must show
CASES = {}
for _mw in (50.0, 10000.0, 1e30):
    for _cw in (1, 0):
        CASES[f"prior/mw{_mw:g}_cw{_cw}"] = dict(
            voxel=ROOM_VS, cfg=dict(default_truncation_distance=ROOM_T, max_weight=_mw, use_const_weight=_cw),
            scans=_room, prior=True, paths=["long_runs"])
CASES["extreme_z/minray0"] = dict(voxel=0.1, cfg=dict(default_truncation_distance=0.4, max_ray_length_m=10.0,
                                                      min_ray_length_m=0.0),
                                  scans=_lidar_extreme_z, prior=False, paths=[], refold=True)
CASES["extreme_z/minray0.1"] = dict(voxel=0.1, cfg=dict(default_truncation_distance=0.4, max_ray_length_m=10.0),
                                    scans=_lidar_extreme_z, prior=False, paths=[], refold=True)
for _shape in ("short", "late_live", "alternating", "clearing"):
    CASES[f"refold/{_shape}"] = dict(voxel=0.1, cfg=dict(default_truncation_distance=0.4),
                                     scans=lambda s=_shape: _refold_cluster(s), prior=False, paths=[], refold=True)
for _f in (1.0, 0.5):
    CASES[f"trunc/c1_wall_x{_f:g}"] = dict(voxel=0.2, cfg=dict(default_truncation_distance=0.2 * _f),
                                           scans=lambda: [scenes.c1_planar_wall()], prior=False, paths=[])
    CASES[f"trunc/room_x{_f:g}"] = dict(voxel=ROOM_VS, cfg=dict(default_truncation_distance=ROOM_VS * _f),
                                        scans=_room, prior=False, paths=["long_runs"])
CASES["max_weight/1e-07"] = dict(voxel=ROOM_VS, cfg=dict(default_truncation_distance=ROOM_T, max_weight=1e-7),
                                 scans=_room, prior=False, paths=["long_runs"], no_paths=["long_rested"])
CASES["max_weight/1"] = dict(voxel=ROOM_VS, cfg=dict(default_truncation_distance=ROOM_T, max_weight=1.0,
                                                     use_const_weight=1),
                             scans=_room, prior=False, paths=["long_runs", "long_rested"])
CASES["max_weight/1e+30"] = dict(voxel=ROOM_VS, cfg=dict(default_truncation_distance=ROOM_T, max_weight=1e30),
                                 scans=_room, prior=False, paths=["long_runs"])
KINDS = (1, 2)
PIN_KEYS = [f"{key}/{kind}" for key in CASES for kind in KINDS]


def _prior_blocks(lib, case):
    """The map after the first scan (integrated by `lib`), mutated: [(block index, serialised words)]."""
    base = po.OracleMap(lib, po.TsdfConfig(integrator_threads=1, **case["cfg"]), case["voxel"], 16)
    base.integrate(2, case["scans"]()[0])
    T, mw = case["cfg"]["default_truncation_distance"], case["cfg"]["max_weight"]
    return [(i, _mutate_prior(base.serialize_block(i, 0), T, mw, seed=k))
            for k, i in enumerate(base.block_indices())]


def reference_side(pin_key, lib):
    """(prior blocks: [(index, serialised words, voxels and updated bits as the oracle holds them after
    deserialising)], scans to integrate, oracle map after them, digest of that map) for `key/kind`."""
    key, kind = pin_key.rsplit("/", 1)
    case = CASES[key]
    scans = case["scans"]()
    prior = _prior_blocks(lib, case) if case["prior"] else []
    if case["prior"]:
        scans = scans[1:]
    omap = po.OracleMap(lib, po.TsdfConfig(integrator_threads=1, **case["cfg"]), case["voxel"], 16)
    for i, words in prior:
        omap.deserialize_block(i, words, 0)
    start = [(i, words) + tuple(omap.block(i)) for i, words in prior]
    for s in scans:
        omap.integrate(int(kind), s)
    return start, scans, omap, pins.map_digest(omap)


@pytest.mark.parametrize("pin_key", PIN_KEYS)
def test_edges_bit_exact_against_reference(pin_key):
    key, kind = pin_key.rsplit("/", 1)
    case = CASES[key]
    prior, scans, omap, digest = reference_side(pin_key, pins.lib())
    pins.check(f"tsdf_edges/{pin_key}", digest)
    cfg = vb.TsdfIntegratorConfig(integrator_threads=1, **case["cfg"])
    layer = vb.Layer(case["voxel"], 16)
    integ = vb.TsdfIntegratorFactory.create(int(kind), cfg, layer)
    integ.countApplyPaths(True)
    ocheck = po.OracleMap(po.OracleLib("port"), po.TsdfConfig(integrator_threads=1, **case["cfg"]), case["voxel"], 16)
    if prior:
        # the voxels and updated() bits the oracle holds after deserialising, inserted as they are
        idx = np.array([p[0] for p in prior], np.int32).reshape(-1, 3)
        vox = np.stack([p[2] for p in prior])
        upd = np.array([p[3] for p in prior], np.uint8)
        layer.insertBlocks(idx, vox, upd)
        for i, words, _, _ in prior:
            ocheck.deserialize_block(i, words, 0)
    seen = {k: 0 for k in vb.api.TsdfIntegratorBase.APPLY_PATHS}
    refolded = 0
    for s in scans:
        integ.integratePointCloud((s[2], s[3]), s[0], s[1])
        ocheck.integrate(int(kind), s)
        gc, oc = integ.counters(), ocheck.counters()
        for k in ("rays", "clear_rays", "updates", "voxels_touched", "blocks_touched", "blocks_allocated"):
            assert gc[k] == oc[k], (k, gc, oc)
        refolded += gc["refolded_bundles"]
        for k, v in integ.applyPaths().items():
            seen[k] += v
    rep = compare_tsdf(layer, omap)
    print(pin_key, rep, "apply paths:", seen, "refolded bundles:", refolded)
    assert rep["blocks_equal"] and rep["observed_equal"] and rep["updated_equal"], rep
    assert rep["color_mismatch"] == 0, rep
    assert rep["n_bit_exact"] == rep["n_voxels"], rep
    gi = layer.getAllAllocatedBlocks()
    gv, _ = layer.getBlocks(gi)
    ov = np.stack([omap.block(i)[0] for i in omap.block_indices()])
    assert np.ascontiguousarray(gv).tobytes() == np.ascontiguousarray(ov).tobytes()   # -0.0 and every colour byte too
    for k in case["paths"]:
        assert seen[k] > 0, (k, seen)
    for k in case.get("no_paths", ()):
        assert seen[k] == 0, (k, seen)
    if case.get("refold") and kind == "2":
        assert refolded > 0, refolded
