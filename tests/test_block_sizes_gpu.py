"""-m gpu: the map at every block size vbx_create accepts below the default (voxels_per_side 1, 2, 4), and
with more than 65,535 blocks, against the reference.

Much of the engine is written in terms of L = log2(voxels_per_side): the update-record key (touched id <<
3L | voxel), the touched-id capacity, the walk's block runs, the mesher's border cubes (at vps 1 every cube
reads up to seven neighbour blocks), the ESDF's one-voxel staging path and the block transfer kernels
(a one-voxel TSDF block is 12 B, an ESDF block 20 B: neither is a multiple of 16 B).  At small block sizes
a scan touches ten to a thousand times more blocks, and a map of two lidar scans at vps 2 holds ~228 k of
them -- more than the 65,535 a grid's y dimension can number.

The exact cases (TSDF, mesh, one-thread ICP) compare with the reference's own library where oracle/_ref
was built, else with the restatement held to the reference's recorded digests (tests/golden/reference_pins.py)."""
import numpy as np
import pytest

import voxblox_b200 as vb
from oracle import pyoracle as po
from tests.golden import reference_pins as pins
from tests.parity import compare_esdf, compare_tsdf
from tests.test_esdf_gpu import EKW, _wall_scans
from tests.test_icp_gpu import PERTURBATIONS, TOL, _close, _perturbed
from tests.test_mesh_gpu import _compare as compare_mesh
from tests.test_tsdf_gpu import _assert_parity
from voxblox_b200 import scenes, sharded

pytestmark = pytest.mark.gpu

KINDS = {"simple": po.SIMPLE, "merged": po.MERGED}
SMALL_VPS = (1, 2, 4)
# pools sized for the cases below (the room scans make ~50 k blocks at vps 1)
MAX_BLOCKS = {1: 1 << 16, 2: 1 << 19, 4: 1 << 17}
COUNTERS = ("rays", "clear_rays", "updates", "voxels_touched", "blocks_touched", "blocks_allocated")


def _room_scans(n=3, width=320, height=240):
    return list(scenes.c3_room_sequence(n_scans=n, width=width, height=height))


SCENES = {
    "room": dict(voxel=0.05, trunc=0.2, scans=_room_scans, cfg={}),
    "c2": dict(voxel=0.1, trunc=0.4, scans=lambda: [scenes.c2_sphere_scan(i, width=320, height=240) for i in range(3)],
               cfg={}),
    "c5": dict(voxel=0.05, trunc=0.2, scans=lambda: [scenes.c5_lidar_scan(i) for i in range(2)],
               cfg=dict(max_ray_length_m=10.0, use_const_weight=1)),
}


def _opts(vps, **kw):
    return vb.EngineOptions(**dict(dict(max_blocks=MAX_BLOCKS[vps]), **kw))


def _tsdf_case(key):
    scene, kind, vps = key.split("/")
    return SCENES[scene], kind, int(vps[3:])


def reference_side(key, lib):
    """The oracle side of case `key`: "tsdf/<scene>/<kind>/vps<v>" -> (scans, map, digest of the map, counters
    after each scan); "mesh/<mode>/<color>/<min weight>/vps<v>" -> (scans, map, digest of the map's meshes, None);
    "icp/vps<v>" -> (scans, map, {"map": digest, "icp": refined poses}, None)."""
    what, rest = key.split("/", 1)
    if what == "tsdf":
        sc, kind, vps = _tsdf_case(rest)
        scans = sc["scans"]()
        omap = po.OracleMap(lib, po.TsdfConfig(default_truncation_distance=sc["trunc"], integrator_threads=1, **sc["cfg"]),
                            sc["voxel"], vps)
        counts = []
        for s in scans:
            omap.integrate(KINDS[kind], s)
            counts.append(omap.counters())
        return scans, omap, pins.map_digest(omap), counts
    if what == "mesh":
        mode, color, min_weight, vps = rest.split("/")
        scans = _room_scans(3, 160, 120)
        omap = po.OracleMap(lib, po.TsdfConfig(default_truncation_distance=0.4, integrator_threads=1), 0.1, int(vps[3:]))
        for s in scans:
            omap.integrate(po.MERGED, s)
            if mode == "incremental":
                omap.mesh_generate(color == "color", float(min_weight), True, True)
        if mode == "full":
            omap.mesh_generate(color == "color", float(min_weight), False, True)
        parts = [omap.mesh_block_indices()]
        for i in parts[0]:
            v, n, c, upd = omap.mesh_block(i)
            parts += [v, n, np.zeros((0, 4), np.uint8) if c is None else c, np.array([upd], np.int32)]
        return scans, omap, pins.array_digest(*parts), None
    vps = int(rest[3:])
    scans = _room_scans(4)
    omap = po.OracleMap(lib, po.TsdfConfig(default_truncation_distance=0.2, integrator_threads=1), 0.05, vps)
    for s in scans[:3]:
        omap.integrate(po.MERGED, s)
    icp = []
    for k, (dt, yaw) in enumerate(PERTURBATIONS):
        q0, t0 = _perturbed(scans[3], dt, yaw)
        q, t, n = omap.icp(po.IcpConfig(), scans[3][0], q0, t0, 7 + k)
        icp.append({"q_wxyz": [float(v).hex() for v in q], "t": [float(v).hex() for v in t], "num_updates": int(n)})
    return scans, omap, {"map": pins.map_digest(omap), "icp": icp}, None


TSDF_KEYS = [f"{sc}/{kind}/vps{v}" for sc in ("room", "c2") for kind in KINDS for v in SMALL_VPS] + ["c5/merged/vps2"]
MESH_KEYS = [f"{mode}/{color}/{w}/vps{v}" for mode in ("incremental", "full") for color in ("color", "nocolor")
             for w in ("0.0001", "0.5") for v in SMALL_VPS]
ICP_VPS = (2, 4)
PIN_KEYS = ([f"tsdf/{k}" for k in TSDF_KEYS] + [f"mesh/{k}" for k in MESH_KEYS] + [f"icp/vps{v}" for v in ICP_VPS])


def _device_tsdf(key, counts):
    """The device's map of TSDF case `key`, its per-scan counters held to `counts` (the restatement's: the
    reference's library reports none)."""
    sc, kind, vps = _tsdf_case(key)
    layer = vb.Layer(sc["voxel"], vps, engine_options=_opts(vps, max_points_per_scan=1 << 19))
    cfg = vb.TsdfIntegratorConfig(default_truncation_distance=sc["trunc"], integrator_threads=1, **sc["cfg"])
    integ = vb.TsdfIntegratorFactory.create(kind, cfg, layer)
    for s, oc in zip(sc["scans"](), counts):
        integ.integratePointCloud((s[2], s[3]), s[0], s[1])
        gc = integ.counters()
        for k in COUNTERS:
            assert gc[k] == oc[k], (key, k, gc, oc)
    return layer


def _pinned(key):
    """reference_side of pinned case `key` with the oracle in use, its digest held to the reference's, and
    the restatement's per-scan counters."""
    lib = pins.lib()
    scans, omap, digest, counts = reference_side(key, lib)
    pins.check(f"block_sizes/{key}", digest)
    if counts is not None and lib.which != "port":
        counts = reference_side(key, po.OracleLib("port"))[3]
    return scans, omap, counts


@pytest.mark.parametrize("key", [k for k in TSDF_KEYS if not k.startswith("c5")])
def test_tsdf_bit_exact_at_small_block_sizes(key):
    """Simple and Merged at one integrator thread: every voxel, the block set, the updated bits and the
    per-scan counters equal the reference's."""
    _, omap, counts = _pinned(f"tsdf/{key}")
    layer = _device_tsdf(key, counts)
    rep = compare_tsdf(layer, omap)
    print(key, rep)
    _assert_parity(rep)


def _layer_bytes(layer):
    idx = layer.getAllAllocatedBlocks()
    vox, upd = layer.getBlocks(idx)
    return idx.tobytes(), vox.tobytes(), np.asarray(upd).tobytes()


@pytest.mark.parametrize("kind", list(KINDS))
@pytest.mark.parametrize("vps", [1, 2])
def test_pipelined_equals_synchronous_at_small_block_sizes(vps, kind):
    """Scans that touch tens of thousands of blocks each through the captured graphs and their grid hints."""
    cfg = vb.TsdfIntegratorConfig(default_truncation_distance=0.2, integrator_threads=1)
    la, ls = vb.Layer(0.05, vps, engine_options=_opts(vps)), vb.Layer(0.05, vps, engine_options=_opts(vps))
    ia, isync = vb.TsdfIntegratorFactory.create(kind, cfg, la), vb.TsdfIntegratorFactory.create(kind, cfg, ls)
    keep = []
    for s in _room_scans(5):
        isync.integratePointCloud((s[2], s[3]), s[0], s[1])
        p, c = np.ascontiguousarray(s[0]), np.ascontiguousarray(s[1])
        keep.append((p, c))
        ia.integratePointCloudAsync((s[2], s[3]), p, c)
    la.sync()
    assert ls.getNumberOfAllocatedBlocks() > 5000
    assert _layer_bytes(la) == _layer_bytes(ls)
    assert ia.counters()["kernel_launches"] == isync.counters()["kernel_launches"] + 1


def _assert_transfers_reproduce(layer, cfg, vps, tmp_path, esdf=None):
    """mirrorUpdated, serializeUpdated, saveToFile -> loadBlocksFromFile and insertSerializedBlocks into fresh
    layers all reproduce what the per-block download (getBlocks) returns; the ESDF layer too when given."""
    idx = layer.getAllAllocatedBlocks()
    vox, upd = layer.getBlocks(idx)
    midx, mvox, mupd = layer.mirrorUpdated(0, 0)
    assert midx.tobytes() == idx.tobytes() and mvox.tobytes() == vox.tobytes()
    assert np.asarray(mupd).tobytes() == np.asarray(upd).tobytes()
    sidx, words, supd = layer.serializeUpdated(0, 0)
    assert sidx.tobytes() == idx.tobytes() and np.asarray(supd).tobytes() == np.asarray(upd).tobytes()
    # block.cc:159-183: distance bits, weight bits, the colour word a | b << 8 | g << 16 | r << 24
    w = words.reshape(len(idx), -1, 3)
    assert w[..., 0].tobytes() == np.ascontiguousarray(vox["distance"]).view(np.uint32).tobytes()
    assert w[..., 1].tobytes() == np.ascontiguousarray(vox["weight"]).view(np.uint32).tobytes()
    col = vox["color"].astype(np.uint32)
    assert (w[..., 2] == (col[..., 3] | col[..., 2] << 8 | col[..., 1] << 16 | col[..., 0] << 24)).all()
    if esdf is not None:
        eidx = esdf.getAllAllocatedBlocks()
        evox, _ = esdf.getBlocks(eidx)
        a, b, _ = esdf.mirrorUpdated(0, 0)
        assert a.tobytes() == eidx.tobytes() and b.tobytes() == evox.tobytes()
        eidx2, ewords, _ = esdf.serializeUpdated(0, 0)
        assert eidx2.tobytes() == eidx.tobytes()
    path = str(tmp_path / f"map_vps{vps}.vxblx")
    assert layer.saveToFile(path, True)
    if esdf is not None:
        assert esdf.saveToFile(path, False)

    def fresh():
        nl = vb.Layer(layer.voxel_size(), vps, engine_options=_opts(vps, max_points_per_scan=max(1 << 19, len(idx))))
        vb.TsdfIntegratorFactory.create("merged", cfg, nl)
        ne = None
        if esdf is not None:
            ne = vb.Layer(layer.voxel_size(), vps, voxel_type="esdf")
            vb.EsdfIntegrator(vb.EsdfIntegratorConfig(), nl, ne)
        return nl, ne
    loaded, loaded_e = fresh()
    assert loaded.loadBlocksFromFile(path) == len(idx)
    assert loaded.getAllAllocatedBlocks().tobytes() == idx.tobytes()
    assert loaded.getBlocks(idx)[0].tobytes() == vox.tobytes()
    if esdf is not None:
        assert loaded_e.loadBlocksFromFile(path) == len(eidx)
        assert loaded_e.serializeUpdated(0, 0)[1].tobytes() == ewords.tobytes()
    des, des_e = fresh()
    des.insertSerializedBlocks(sidx, words, supd)
    assert des.getAllAllocatedBlocks().tobytes() == idx.tobytes()
    got, gupd = des.getBlocks(idx)
    assert got.tobytes() == vox.tobytes() and np.asarray(gupd).tobytes() == np.asarray(upd).tobytes()
    if esdf is not None:
        des_e.insertSerializedBlocks(eidx, ewords)
        assert des_e.serializeUpdated(0, 0)[1].tobytes() == ewords.tobytes()


@pytest.mark.parametrize("vps", [1, 2, 4])
def test_block_transfers_at_small_block_sizes(vps, tmp_path):
    """A one-voxel TSDF block is 12 B and an ESDF block 20 B: the mirror, the serialiser and the file
    round trip work on payloads that are not a multiple of 16 B."""
    cfg = vb.TsdfIntegratorConfig(default_truncation_distance=0.4, integrator_threads=1)
    layer = vb.Layer(0.1, vps, engine_options=_opts(vps))
    integ = vb.TsdfIntegratorFactory.create("merged", cfg, layer)
    esdf = vb.Layer(0.1, vps, voxel_type="esdf")
    eint = vb.EsdfIntegrator(vb.EsdfIntegratorConfig(min_distance_m=0.2), layer, esdf)
    for s in _room_scans(2, 96, 72):
        integ.integratePointCloud((s[2], s[3]), s[0], s[1])
    eint.updateFromTsdfLayer(True)
    assert esdf.getNumberOfAllocatedBlocks() > 0
    _assert_transfers_reproduce(layer, cfg, vps, tmp_path, esdf)
    # the mirror's clear mask still clears exactly the mirrored bit
    want = layer.getAllUpdatedBlocks(1)
    idx, _, _ = layer.mirrorUpdated(2, 2)
    assert idx.tobytes() == want.tobytes() and layer.getAllUpdatedBlocks(1).shape[0] == 0


def test_more_than_65535_integrated_blocks(tmp_path):
    """C5 (two lidar scans) at vps 2 makes ~228 k blocks: bit-exact against the reference, then every block
    transfer path reproduces the per-block download."""
    key = "c5/merged/vps2"
    _, omap, counts = _pinned(f"tsdf/{key}")
    layer = _device_tsdf(key, counts)
    assert layer.getNumberOfAllocatedBlocks() > 65535
    rep = compare_tsdf(layer, omap)
    print(key, rep)
    _assert_parity(rep)
    sc, _, _ = _tsdf_case(key)
    cfg = vb.TsdfIntegratorConfig(default_truncation_distance=sc["trunc"], integrator_threads=1, **sc["cfg"])
    _assert_transfers_reproduce(layer, cfg, 2, tmp_path)


def test_more_than_65535_uploaded_blocks(tmp_path):
    """70,000 blocks of seeded random voxels at vps 4 into both layers in one upload, round-tripped through
    getBlocks, serializeUpdated, insertSerializedBlocks and a .vxblx file; a sample of the serialised blocks
    is compared word for word with the oracle's serializeToIntegers of the same voxels."""
    vps, n = 4, 70000
    nv = vps ** 3
    rng = np.random.default_rng(11)
    idx = np.unique(rng.integers(-300, 300, (n + 4000, 3), dtype=np.int32), axis=0)
    idx = idx[rng.permutation(len(idx))[:n]]
    assert len(idx) == n
    tv = np.zeros((n, nv), vb.TSDF_DTYPE)
    tv["distance"] = rng.uniform(-0.4, 0.4, (n, nv)).astype(np.float32)
    tv["weight"] = rng.uniform(0.0, 9.0, (n, nv)).astype(np.float32)
    tv["color"] = rng.integers(0, 256, (n, nv, 4), dtype=np.uint8)
    tupd = rng.integers(0, 8, n).astype(np.uint8)
    ev = np.zeros((n, nv), vb.ESDF_DTYPE)
    ev["distance"] = rng.uniform(-2.0, 2.0, (n, nv)).astype(np.float32)
    for f in ("observed", "hallucinated", "in_queue", "fixed"):
        ev[f] = rng.integers(0, 2, (n, nv), dtype=np.uint8)
    ev["parent"] = rng.integers(-128, 128, (n, nv, 3), dtype=np.int32)
    opts = vb.EngineOptions(max_blocks=1 << 17, max_points_per_scan=1 << 17)
    cfg = vb.TsdfIntegratorConfig(default_truncation_distance=0.4, integrator_threads=1)

    def fresh():
        layer = vb.Layer(0.1, vps, engine_options=opts)
        vb.TsdfIntegratorFactory.create("merged", cfg, layer)
        esdf = vb.Layer(0.1, vps, voxel_type="esdf")
        vb.EsdfIntegrator(vb.EsdfIntegratorConfig(), layer, esdf)
        return layer, esdf
    layer, esdf = fresh()
    layer.insertBlocks(idx, tv, tupd)
    esdf.insertBlocks(idx, ev)
    order = np.lexsort((idx[:, 2], idx[:, 1], idx[:, 0]))
    sidx = idx[order]
    assert layer.getAllAllocatedBlocks().tobytes() == sidx.tobytes()
    assert esdf.getAllAllocatedBlocks().tobytes() == sidx.tobytes()
    got, gupd = layer.getBlocks(idx)
    assert got.tobytes() == tv.tobytes() and gupd.tobytes() == tupd.tobytes()
    assert esdf.getBlocks(idx)[0].tobytes() == ev.tobytes()
    _assert_transfers_reproduce(layer, cfg, vps, tmp_path, esdf)
    # the device's words for a sample of blocks equal the oracle's serialisation of the same voxels
    words = layer.serializeUpdated(0, 0)[1]
    ewords = esdf.serializeUpdated(0, 0)[1]
    scratch = po.OracleMap(po.OracleLib("port"), po.TsdfConfig(default_truncation_distance=0.4), 0.1, vps)
    scratch.esdf_create(po.EsdfConfig())
    for k in list(range(0, n, 997)) + [65534, 65535, 65536, n - 1]:
        i = sidx[k]
        j = order[k]
        scratch.deserialize_block(i, words[k], 0)
        assert scratch.block(i, 0)[0].tobytes() == tv[j].tobytes(), tuple(i)
        assert scratch.serialize_block(i, 0).tobytes() == words[k].tobytes(), tuple(i)
        # ESDF words are lossy (serializeDirection sign-extends a negative y or z over the bytes above it):
        # the oracle's re-encoding of what it decodes is a fixed point, and block.cc:8-41,203-234 restated
        # on the uploaded voxels gives the same words
        scratch.deserialize_block(i, ewords[k], 1)
        assert scratch.serialize_block(i, 1).tobytes() == ewords[k].tobytes(), tuple(i)
        par = ev[j]["parent"].astype(np.int64)
        w2 = ((par[:, 0] << 24) | (par[:, 1] << 16) | (par[:, 2] << 8)) & 0xFFFFFFFF
        w2 |= (ev[j]["observed"] != 0) * 1 | (ev[j]["hallucinated"] != 0) * 2 | (ev[j]["in_queue"] != 0) * 4 | \
            (ev[j]["fixed"] != 0) * 8
        want = np.stack([ev[j]["distance"].view(np.uint32), w2.astype(np.uint32)], axis=1).reshape(-1)
        assert want.tobytes() == ewords[k].tobytes(), tuple(i)


@pytest.mark.parametrize("key", MESH_KEYS)
def test_mesh_at_small_block_sizes(key):
    """The mesher against the reference's MeshIntegrator: at vps 1 every cube is a border cube reading up to
    seven neighbour blocks."""
    mode, color, min_weight, vps = key.split("/")
    vps = int(vps[3:])
    scans, omap, _ = _pinned(f"mesh/{key}")
    layer = vb.Layer(0.1, vps, engine_options=_opts(vps))
    integ = vb.TsdfIntegratorFactory.create(
        "merged", vb.TsdfIntegratorConfig(default_truncation_distance=0.4, integrator_threads=1), layer)
    mesh_layer = vb.MeshLayer(layer.block_size())
    mesher = vb.MeshIntegrator(vb.MeshIntegratorConfig(use_color=color == "color", min_weight=float(min_weight)),
                               layer, mesh_layer)
    for s in scans:
        integ.integratePointCloud((s[2], s[3]), s[0], s[1])
        if mode == "incremental":
            mesher.generateMesh(True, True)
    if mode == "full":
        mesher.generateMesh(False, True)
    assert compare_tsdf(layer, omap)["max_rel_err"] == 0.0       # (incl. the updated bits)
    rep = compare_mesh(mesh_layer, omap)
    print(key, rep)
    assert rep["vertices"] > 1000
    assert rep["count_mismatch"] == 0 and rep["vertex_mismatch"] == 0 and rep["normal_mismatch"] == 0, rep
    assert rep["color_mismatch"] == 0, rep


def _esdf_setup(vps, ekw):
    cfg = vb.TsdfIntegratorConfig(default_truncation_distance=0.4, integrator_threads=1)
    tsdf = vb.Layer(0.1, vps, engine_options=_opts(vps))
    integ = vb.TsdfIntegratorFactory.create("merged", cfg, tsdf)
    esdf = vb.Layer(0.1, vps, voxel_type="esdf")
    eint = vb.EsdfIntegrator(vb.EsdfIntegratorConfig(**ekw), tsdf, esdf)
    omap = po.OracleMap(po.OracleLib("port"), po.TsdfConfig(default_truncation_distance=0.4), 0.1, vps)
    omap.esdf_create(po.EsdfConfig(**ekw))
    return tsdf, integ, esdf, eint, omap


@pytest.mark.parametrize("vps", [1, 2])
def test_esdf_incremental_at_small_block_sizes(vps):
    """As test_esdf_other_block_sizes; at vps 1 the propagation stages its neighbours without bulk copies."""
    tsdf, integ, esdf, eint, omap = _esdf_setup(vps, EKW)
    for s in _wall_scans():
        integ.integratePointCloud((s[2], s[3]), s[0], s[1])
        omap.integrate(2, s, order=po.ORDER_REFERENCE)
        eint.updateFromTsdfLayer(True)
        omap.esdf_update(batch=False, clear_updated_flag=True)
    rep = compare_esdf(esdf, omap, 4.0)
    print("vps", vps, rep)
    assert rep["blocks_equal"] and rep["observed_equal"] and rep["fixed_equal"], rep
    assert rep["n_bit_exact"] >= 0.995 * rep["voxels_observed"], rep


@pytest.mark.parametrize("vps", [1, 2])
def test_esdf_batch_at_small_block_sizes(vps):
    """As test_esdf_batch_matches_oracle, on the same room scans."""
    tsdf, integ, esdf, eint, omap = _esdf_setup(vps, EKW)
    for s in scenes.c3_room_sequence(n_scans=4, width=160, height=120):
        integ.integratePointCloud((s[2], s[3]), s[0], s[1])
        omap.integrate(2, s, order=po.ORDER_REFERENCE)
    assert compare_tsdf(tsdf, omap)["max_rel_err"] == 0.0
    eint.updateFromTsdfLayerBatch()
    omap.esdf_update(batch=True)
    rep = compare_esdf(esdf, omap, 4.0)
    print("vps", vps, rep)
    assert rep["blocks_equal"] and rep["observed_equal"] and rep["fixed_equal"], rep
    assert rep["flag_bytes_clean"] and rep["in_queue_gpu"] == 0, rep
    assert rep["n_bit_exact"] >= 0.93 * rep["voxels_observed"], rep
    assert rep["rmse"] < 0.1 * 0.1, rep
    assert rep["max_abs_err"] <= 2 * 0.1 * 3 ** 0.5, rep


def _icp_layer(vps, scans, omap):
    layer = vb.Layer(0.05, vps, engine_options=_opts(vps))
    integ = vb.TsdfIntegratorFactory.create(
        "merged", vb.TsdfIntegratorConfig(default_truncation_distance=0.2, integrator_threads=1), layer)
    for s in scans:
        integ.integratePointCloud((s[2], s[3]), s[0], s[1])
    rep = compare_tsdf(layer, omap)
    assert rep["blocks_equal"] and rep["n_bit_exact"] == rep["n_voxels"], rep
    return layer


def _assert_icp_close(rep):
    assert rep["dq"] <= TOL and rep["dt_rel"] <= TOL, rep
    assert abs(rep["updates"][0] - rep["updates"][1]) <= max(2, rep["updates"][1] // 1000), rep


@pytest.mark.parametrize("vps", ICP_VPS)
def test_icp_one_thread_at_small_block_sizes(vps):
    """At vps 2 nearly every interpolation crosses a block boundary."""
    key = f"icp/vps{vps}"
    scans, omap, got, _ = reference_side(key, pins.lib())
    want = pins.recorded(f"block_sizes/{key}")
    assert got["map"] == want["map"], "the oracle's map is not the reference's"
    layer = _icp_layer(vps, scans[:3], omap)
    for k, (dt, yaw) in enumerate(PERTURBATIONS):
        q0, t0 = _perturbed(scans[3], dt, yaw)
        dev = vb.ICP(vb.ICPConfig()).runICP(layer, scans[3][0], (q0, t0), seed=7 + k)
        r = want["icp"][k]
        ref = (np.array([float.fromhex(v) for v in r["q_wxyz"]]), np.array([float.fromhex(v) for v in r["t"]]),
               r["num_updates"])
        rep = _close(dev, ref)
        print("vps", vps, "perturbation", dt, yaw, rep)
        _assert_icp_close(rep)


@pytest.mark.parametrize("threads", [4, 32])
@pytest.mark.parametrize("vps", ICP_VPS)
def test_icp_round_robin_threads_at_small_block_sizes(vps, threads):
    scans = _room_scans(4)
    omap = po.OracleMap(po.OracleLib("port"), po.TsdfConfig(default_truncation_distance=0.2, integrator_threads=1),
                        0.05, vps)
    for s in scans[:3]:
        omap.integrate(po.MERGED, s)
    layer = _icp_layer(vps, scans[:3], omap)
    q0, t0 = _perturbed(scans[3], (0.05, -0.04, 0.02), 0.01)
    for mb, ratio in ((20, 0.8), (50, 0.5)):
        cfg = dict(num_threads=threads, mini_batch_size=mb, min_match_ratio=ratio, subsample_keep_ratio=0.7)
        dev = vb.ICP(vb.ICPConfig(**cfg)).runICP(layer, scans[3][0], (q0, t0), seed=123)
        rep = _close(dev, omap.icp(po.IcpConfig(**cfg), scans[3][0], q0, t0, 123))
        print("vps", vps, "threads", threads, "mini batch", mb, rep)
        _assert_icp_close(rep)


@pytest.mark.parametrize("kind", ["merged", "simple"])
def test_union_of_shards_at_vps2(kind):
    """W = 2 shards on one GPU: together they hold exactly the single-GPU map's blocks, bit for bit."""
    world, vps = 2, 2
    cfg = vb.TsdfIntegratorConfig(default_truncation_distance=0.4, integrator_threads=1)
    scans = scenes.c3_room_sequence(n_scans=3, width=160, height=120)
    full = vb.Layer(0.1, vps, engine_options=_opts(vps))
    fi = vb.TsdfIntegratorFactory.create(kind, cfg, full)
    for s in scans:
        fi.integratePointCloud((s[2], s[3]), s[0], s[1])
    full_blocks = full.blocks()
    seen = {}
    for rank in range(world):
        layer = vb.Layer(0.1, vps, engine_options=sharded.shard_options(rank, world, max_blocks=MAX_BLOCKS[vps]))
        integ = vb.TsdfIntegratorFactory.create(kind, cfg, layer)
        for s in scans:
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
