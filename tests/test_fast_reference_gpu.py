"""-m gpu: the Fast integrator against the reference's one-thread FastTsdfIntegrator, voxel for voxel.

Fast consults two approximate sets (ApproxHashSet, utils/approx_hash_array.h) while it walks: a start-cell
set that drops a ray whose start cell an earlier ray already used, and an observed-voxel set that stops a
ray after more than max_consecutive_ray_collisions voxels in a row that earlier rays already walked.  At
one integrator thread the reference consults them in point order and is deterministic; on the device the
rays of one call race for them.  So the map is compared exactly wherever the device's schedule cannot
matter:
  * serial: vbx_debug_serial_fast walks the rays on one device thread in point order, the reference's
    schedule, at the default config and its variants;
  * parallel: the normal launch with a start grid so fine that no two points share a start cell and no
    cut-off (max_consecutive_ray_collisions = 2^31 - 1), so every ray is cast on both sides -- each case
    first proves that from the counters -- through the pass splitting, asynchronous submission, every
    block size and shards;
  * collisions: the normal launch on calls of a few axis-aligned rays that share no voxel but the sensor's
    own (with one colour and one range, so whichever ray reaches it first makes the same update), over
    the cut-off thresholds and reset cadences, with repeated points and rays extended along earlier ones.

Every case compares distance, weight, colour, the block set and the updated bits, and holds the per-scan
counters to the restatement's (the reference's library reports none).  The comparison is with the
reference's own library where oracle/_ref was built, else with the restatement held to the reference's
recorded digests (tests/golden/reference_pins.py).

The reference keeps the reset counter of clear_checks_every_n_frames in a function-level static shared by
every Fast integrator of the process (tsdf_integrator.cc:564); the engine keeps one per map.  Each oracle
run first zeroes that static (prime), so the oracle's map starts where a fresh engine map does."""
import numpy as np
import pytest

import voxblox_b200 as vb
from oracle import pyoracle as po
from tests.golden import reference_pins as pins
from tests.parity import compare_tsdf
from tests.test_tsdf_gpu import _assert_parity
from voxblox_b200 import scenes, sharded

pytestmark = pytest.mark.gpu

COUNTERS = ("rays", "clear_rays", "updates", "voxels_touched", "blocks_touched", "blocks_allocated")
IDENTITY = np.array([1.0, 0.0, 0.0, 0.0], np.float32)
NEVER_CUT = 2 ** 31 - 1


def _room(n, w, h):
    return list(scenes.c3_room_sequence(n_scans=n, width=w, height=h))


SCENES = {
    "c1": dict(voxel=0.2, trunc=0.8, scans=lambda: [scenes.c1_planar_wall()]),
    "room": dict(voxel=0.1, trunc=0.4, scans=lambda: _room(4, 160, 120)),
    "room320": dict(voxel=0.05, trunc=0.2, scans=lambda: _room(3, 320, 240)),
    "c2": dict(voxel=0.1, trunc=0.4, scans=lambda: [scenes.c2_sphere_scan(i, width=320, height=240) for i in range(3)]),
    "c3": dict(voxel=0.05, trunc=0.2, scans=lambda: _room(3, 640, 480)),
}

# the config variants of test_tsdf_gpu.py and the Fast integrator's own options (cfg, freespace_points)
VARIANTS = {
    "const_weight": (dict(use_const_weight=1), False),
    "no_carving": (dict(voxel_carving_enabled=0), False),
    "no_dropoff": (dict(use_weight_dropoff=0), False),
    "sparsity": (dict(use_sparsity_compensation_factor=1, sparsity_compensation_factor=3.0), False),
    "max_ray_2": (dict(max_ray_length_m=2.0), False),
    "max_ray_2_no_clear": (dict(max_ray_length_m=2.0, allow_clear=0), False),
    "min_ray_1.5": (dict(min_ray_length_m=1.5), False),
    "max_weight_5": (dict(max_weight=5.0), False),
    "sorted": (dict(integration_order_mode=1), False),
    "freespace": ({}, True),
    "start_1": (dict(start_voxel_subsampling_factor=1.0), False),
    "start_4": (dict(start_voxel_subsampling_factor=4.0), False),
    "collisions_-1": (dict(max_consecutive_ray_collisions=-1), False),
    "collisions_0": (dict(max_consecutive_ray_collisions=0), False),
    "collisions_1": (dict(max_consecutive_ray_collisions=1), False),
    "collisions_5": (dict(max_consecutive_ray_collisions=5), False),
    "clear_every_2": (dict(clear_checks_every_n_frames=2), False),
    "clear_every_3": (dict(clear_checks_every_n_frames=3), False),
}

SERIAL_KEYS = ([f"serial/{sc}/default" for sc in ("c1", "room", "room320", "c2")] +
               [f"serial/room/{v}" for v in VARIANTS])

# the order-independent regime: no cut-off, and a start grid of 1/64 voxel, in which no two points of a room
# scan share a start cell.  A 640x480 scan still has a few pairs of cells whose 32-bit hashes (LongIndexHash)
# are equal; those points are left out of the scan (_distinct_start_cells).
START_FACTOR = 64.0
PARALLEL_CFG = dict(start_voxel_subsampling_factor=START_FACTOR, max_consecutive_ray_collisions=NEVER_CUT)
PARALLEL_VPS = (1, 2, 4, 8, 16)
PARALLEL_KEYS = ["parallel/c3/vps16"] + [f"parallel/room/vps{v}" for v in PARALLEL_VPS]

# ---- calls of a few axis-aligned rays (voxel 0.1): the sensor sits at a voxel centre, so a ray along an
# axis stays in its row of voxels and the rays of one call share the sensor's voxel only
SENSORS = {"origin": (0.05, 0.05, 0.05), "away": (1.35, -0.75, 0.45)}
COLOR = (200, 120, 40, 255)
AXES = [(1, 0, 0), (-1, 0, 0), (0, 1, 0), (0, -1, 0), (0, 0, 1), (0, 0, -1)]


def _call(points_C, t, q=IDENTITY):
    pts = np.array(points_C, np.float32).reshape(-1, 3)
    cols = np.tile(np.array(COLOR, np.uint8), (len(pts), 1))
    return pts, cols, np.asarray(q, np.float32), np.array(t, np.float32)


def _axis_calls(t):
    six = [[1.5 * c for c in ax] for ax in AXES]
    return [
        _call(six[:1], t),                                        # one ray
        _call(six, t),                                            # six rays meeting in the sensor's voxel
        _call([six[0], [-2.5, 0, 0]], t),                         # a repeated point (start cell already used)
        _call([[2.5, 0, 0], [0, 0, -2.2]], t),                   # rays extended along earlier rays
        _call(np.zeros((0, 3)), t),                               # an empty cloud still counts for the cadence
        _call([[0, 2.0, 0], [0, -1.5, 0], [0, 0, 1.9]], t),
        _call(six[::-1], t),                                      # the six again, in the other order
    ]


COLLISION_KEYS = [f"collisions/{s}/max{m}/every{k}" for s in SENSORS for m in (-1, 0, 1, 2) for k in (1, 2, 3)]
# the reference's sets read an unwritten slot as hash 0, the hash of voxel / start cell (0, 0, 0)
FINDING_KEYS = ["finding/origin_voxel/max0", "finding/origin_voxel/max1", "finding/origin_start_cell/inside",
                "finding/origin_start_cell/next"]
TIME_KEYS = ["time/0", "time/nan"]
PIN_KEYS = SERIAL_KEYS + PARALLEL_KEYS + COLLISION_KEYS + FINDING_KEYS + TIME_KEYS


def _distinct_start_cells(scan, voxel):
    """The scan without the points whose start cell's hash another point's start cell also has.  The cells
    are computed here in double precision: near a cell boundary, where the integrators' float arithmetic
    may round the other way, both cells count as the point's."""
    pts, cols, q, t = scan
    x = (pts.astype(np.float64) @ scenes.quat_to_matrix(q).T + t) * (START_FACTOR / voxel)
    x = np.where(np.isfinite(x), x, 0.5)
    lo, hi = np.floor(x - 0.01).astype(np.int64), np.floor(x + 0.01).astype(np.int64)
    cand = []
    for m in range(8):
        g = np.where([(m >> a) & 1 for a in range(3)], hi, lo)
        cand.append((g[:, 0] + g[:, 1] * 17191 + g[:, 2] * 17191 ** 2) & 0xFFFFFFFF)
    cand = np.sort(np.stack(cand, axis=1), axis=1)
    first = np.concatenate([np.ones((len(x), 1), bool), cand[:, 1:] != cand[:, :-1]], axis=1)
    owner = np.repeat(np.arange(len(x)), 8).reshape(-1, 8)[first]
    hashes = cand[first]
    _, inv, cnt = np.unique(hashes, return_inverse=True, return_counts=True)
    shared = np.zeros(len(x), bool)
    shared[owner[cnt[inv.reshape(-1)] > 1]] = True
    return np.ascontiguousarray(pts[~shared]), np.ascontiguousarray(cols[~shared]), q, t


def case(key):
    """key -> dict(voxel, trunc, cfg, freespace, calls, vps)."""
    parts = key.split("/")
    c = dict(cfg={}, freespace=False, vps=16)
    if parts[0] == "serial":
        sc = SCENES[parts[1]]
        c.update(voxel=sc["voxel"], trunc=sc["trunc"], calls=sc["scans"]())
        if parts[2] != "default":
            c["cfg"], c["freespace"] = dict(VARIANTS[parts[2]][0]), VARIANTS[parts[2]][1]
    elif parts[0] == "parallel":
        sc = SCENES[parts[1]]
        c.update(voxel=sc["voxel"], trunc=sc["trunc"], calls=[_distinct_start_cells(s, sc["voxel"]) for s in sc["scans"]()],
                 cfg=dict(PARALLEL_CFG), vps=int(parts[2][3:]))
    elif parts[0] == "collisions":
        c.update(voxel=0.1, trunc=0.4, calls=_axis_calls(SENSORS[parts[1]]),
                 cfg=dict(use_const_weight=1, max_consecutive_ray_collisions=int(parts[2][3:]),
                          clear_checks_every_n_frames=int(parts[3][5:])))
    elif parts[0] == "finding":
        c.update(voxel=0.1, trunc=0.4)
        if parts[1] == "origin_voxel":
            # sensor at the world origin: the ray ends in voxel (0, 0, 0)
            c.update(calls=[_call([[1.0, 0.33, 0.21]], (0, 0, 0))],
                     cfg=dict(max_consecutive_ray_collisions=int(parts[2][3:])))
        else:
            # a point in start cell (0, 0, 0) (0.05 m cells), and one in the next cell
            p = (0.02, 0.02, 0.02) if parts[2] == "inside" else (0.12, 0.02, 0.02)
            c.update(calls=[_call([[p[0] - 1.0, p[1] - 1.0, p[2] - 1.0]], (1, 1, 1))])
    elif parts[0] == "time":
        c.update(voxel=0.1, trunc=0.4, calls=_room(3, 96, 72),
                 cfg=dict(max_integration_time_s=0.0 if parts[1] == "0" else float("nan"),
                          clear_checks_every_n_frames=3))
    else:
        raise KeyError(key)
    return c


def prime(lib):
    """Zero the oracle library's process-wide reset counter: one Fast call with clear_checks_every_n_frames = 1."""
    m = po.OracleMap(lib, po.TsdfConfig(integrator_threads=1, clear_checks_every_n_frames=1), 0.1, 16)
    m.integrate(po.FAST, _call([[1.0, 0.0, 0.0]], (0, 0, 0)))
    m.close()


def reference_side(key, lib):
    """(case, oracle map, digest of the map, counters after each call) of case `key` on `lib`."""
    c = case(key)
    prime(lib)
    omap = po.OracleMap(lib, po.TsdfConfig(default_truncation_distance=c["trunc"], integrator_threads=1, **c["cfg"]),
                        c["voxel"], c["vps"])
    counts = []
    for s in c["calls"]:
        omap.integrate(po.FAST, s, freespace=c["freespace"])
        counts.append(omap.counters())
    return c, omap, pins.map_digest(omap), counts


def _pinned(key):
    """reference_side of `key` with the oracle in use, its digest held to the reference's, and the
    restatement's per-call counters."""
    lib = pins.lib()
    c, omap, digest, counts = reference_side(key, lib)
    pins.check(f"fast_reference/{key}", digest)
    if lib.which != "port":
        counts = reference_side(key, po.OracleLib("port"))[3]
    return c, omap, counts


def _config(c):
    return vb.TsdfIntegratorConfig(default_truncation_distance=c["trunc"], integrator_threads=1, **c["cfg"])


def _layer(c, **opts):
    if c["vps"] < 16:
        opts.setdefault("max_blocks", 1 << 17)
    return vb.Layer(c["voxel"], c["vps"], engine_options=vb.EngineOptions(**opts))


def _device(c, counts, serial=False, counters=COUNTERS, **opts):
    """The device's map of case `c` (one synchronous call per entry), its per-call `counters` held to `counts`."""
    layer = _layer(c, **opts)
    integ = vb.TsdfIntegratorFactory.create("fast", _config(c), layer)
    if serial:
        integ.serialFast(True)
    for k, (s, oc) in enumerate(zip(c["calls"], counts)):
        integ.integratePointCloud((s[2], s[3]), s[0], s[1], freespace_points=c["freespace"])
        gc = integ.counters()
        for name in counters:
            assert gc[name] == oc[name], (k, name, gc, oc)
    return layer, integ


def _layer_bytes(layer):
    idx = layer.getAllAllocatedBlocks()
    vox, upd = layer.getBlocks(idx)
    return idx.tobytes(), vox.tobytes(), np.asarray(upd).tobytes()


# ----------------------------------------------------------------------------- serial launch
@pytest.mark.parametrize("key", SERIAL_KEYS)
def test_serial_launch_matches_reference(key):
    c, omap, counts = _pinned(key)
    layer, _ = _device(c, counts, serial=True, max_points_per_scan=1 << 17)
    rep = compare_tsdf(layer, omap)
    print(key, rep)
    assert rep["voxels_observed"] > 0 or key.endswith("collisions_-1"), rep  # (-1: every ray stops at once)
    _assert_parity(rep)


# ----------------------------------------------------------------------------- parallel launch, no set decision
def _assert_every_ray_cast(counts):
    """The regime holds: the restatement cast a ray for every valid point of every call (no start cell
    shared, no cut-off), so no set decision can have depended on the order."""
    for k, oc in enumerate(counts):
        assert oc["valid_points"] > 0 and oc["rays"] + oc["clear_rays"] == oc["valid_points"], (k, oc)


@pytest.mark.parametrize("key", PARALLEL_KEYS)
def test_parallel_launch_order_independent_regime(key):
    """Full-size C3 and the room stream at every block size.  The device's ray counts (checked per call in
    _device) equal the restatement's, which cast a ray for every valid point."""
    c, omap, counts = _pinned(key)
    _assert_every_ray_cast(counts)
    layer, _ = _device(c, counts, max_points_per_scan=640 * 480)
    rep = compare_tsdf(layer, omap)
    print(key, rep)
    _assert_parity(rep)


def test_parallel_launch_in_passes():
    """More update records than one pass holds: the call is applied in passes and still equals the reference."""
    key = "parallel/room/vps16"
    c, omap, counts = _pinned(key)
    # (voxels_touched counts the distinct voxels of each pass, as in test_tsdf_gpu.py's pass tests)
    layer, integ = _device(c, counts, counters=[k for k in COUNTERS if k != "voxels_touched"],
                           max_updates_per_pass=60000)
    assert integ.counters()["passes"] > 1, integ.counters()
    rep = compare_tsdf(layer, omap)
    print(key, rep, integ.counters())
    _assert_parity(rep)


def test_parallel_launch_async_equals_synchronous():
    """Fast's front half reads its sets, so an asynchronous submission runs synchronously, in order."""
    key = "parallel/room/vps16"
    c, omap, counts = _pinned(key)
    ls, _ = _device(c, counts)
    la = _layer(c)
    ia = vb.TsdfIntegratorFactory.create("fast", _config(c), la)
    keep = []
    for s in c["calls"]:
        p, col = np.ascontiguousarray(s[0]), np.ascontiguousarray(s[1])
        keep.append((p, col))
        ia.integratePointCloudAsync((s[2], s[3]), p, col)
    la.sync()
    assert _layer_bytes(la) == _layer_bytes(ls)
    rep = compare_tsdf(la, omap)
    print(key, rep)
    _assert_parity(rep)


@pytest.mark.parametrize("world", [2, 3])
def test_parallel_launch_union_of_shards(world):
    """Each rank walks every ray through its own sets and creates only the blocks it owns: together the
    shards hold exactly the single map's blocks, and the single map is the reference's."""
    key = "parallel/room/vps16"
    c, omap, counts = _pinned(key)
    full, _ = _device(c, counts)
    _assert_parity(compare_tsdf(full, omap))
    full_blocks = full.blocks()
    seen = {}
    for rank in range(world):
        layer = vb.Layer(c["voxel"], c["vps"], engine_options=sharded.shard_options(rank, world))
        integ = vb.TsdfIntegratorFactory.create("fast", _config(c), layer)
        for s in c["calls"]:
            integ.integratePointCloud((s[2], s[3]), s[0], s[1])
        blocks = layer.blocks()
        idx = np.array(sorted(blocks), np.int32).reshape(-1, 3)
        assert len(idx) and (sharded.block_owner(idx, world) == rank).all(), "a rank created a block it does not own"
        for k, v in blocks.items():
            assert k not in seen
            seen[k] = v
    assert sorted(seen) == sorted(full_blocks)
    for k in full_blocks:
        assert seen[k].tobytes() == full_blocks[k].tobytes(), k


# ----------------------------------------------------------------------------- parallel launch, set decisions
@pytest.mark.parametrize("key", COLLISION_KEYS + FINDING_KEYS)
def test_parallel_launch_deterministic_collisions(key):
    """Cut-offs on voxels observed by earlier calls, start cells used by earlier calls, the reset cadence
    (with an empty call in it), and the sets' treatment of hash 0 (voxel and start cell (0, 0, 0))."""
    c, omap, counts = _pinned(key)
    layer, _ = _device(c, counts)
    rep = compare_tsdf(layer, omap)
    print(key, rep, counts)
    _assert_parity(rep)


@pytest.mark.parametrize("key", TIME_KEYS)
def test_non_positive_integration_time_integrates_nothing(key):
    """The reference checks max_integration_time_s before each point: at 0 or NaN no point is integrated."""
    c, omap, counts = _pinned(key)
    assert all(oc["rays"] == 0 and oc["clear_rays"] == 0 for oc in counts), counts
    layer, _ = _device(c, counts)
    assert layer.getNumberOfAllocatedBlocks() == 0 and len(omap.block_indices()) == 0
