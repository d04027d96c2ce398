"""-m gpu: every integrator's ray walk runs in the front half against the hand-off set's private block table,
and k_assign creates the blocks in submission order.  A table left dirty by an earlier scan of the same set, an
id resolved twice across the passes of one call, or a fallback ray that bypasses the table would give wrong
block ids: wrong voxels, or wrong touched / allocated counts.  Maps are compared bit for bit (distance, weight,
colour, updated bits, block set) with synchronous calls and with the reference's own TsdfIntegrator at one
thread (oracle/_ref) where that library exists, else with the restatement pinned to it; per-call counters with
the restatement (the reference's harness does not count)."""
import numpy as np
import pytest

import voxblox_b200 as vb
from oracle import pyoracle as po
from tests.parity import compare_tsdf
from voxblox_b200 import scenes

pytestmark = pytest.mark.gpu

TRUNC = 0.4
CFG = dict(default_truncation_distance=TRUNC, integrator_threads=1)
COUNTERS = ("rays", "clear_rays", "updates", "voxels_touched", "blocks_touched", "blocks_allocated")


def _layer_bytes(layer):
    idx = layer.getAllAllocatedBlocks()
    vox, upd = layer.getBlocks(idx)
    return idx.tobytes(), vox.tobytes(), np.asarray(upd).tobytes()


def _reference_map(voxel, **cfg):
    which = "reference" if po.available("reference") else "port"
    return po.OracleMap(po.OracleLib(which), po.TsdfConfig(**CFG, **cfg), voxel, 16)


def _port_map(voxel, **cfg):
    return po.OracleMap(po.OracleLib("port"), po.TsdfConfig(**CFG, **cfg), voxel, 16)


def _assert_bit_exact(rep):
    assert rep["blocks_equal"] and rep["observed_equal"] and rep["updated_equal"], rep
    assert rep["color_mismatch"] == 0 and rep["max_rel_err"] == 0.0, rep
    assert rep["n_bit_exact"] == rep["n_voxels"], rep


def _shifted(s, offset):
    """the same scan taken from a sensor moved by offset: a disjoint set of blocks for a large offset"""
    return s[0], s[1], s[2], (np.asarray(s[3], np.float64) + offset).astype(np.float32)


def _alternate_between_disjoint_regions(monkeypatch, kind):
    """Two hand-off sets, reused scan after scan, each seeing every region in turn: the private table of
    a set must be clean when its next scan starts, whatever blocks the previous one met."""
    monkeypatch.setenv("VBX_ASYNC_SETS", "2")
    opts = dict(max_updates_per_pass=1 << 22)
    la = vb.Layer(0.1, 16, engine_options=vb.EngineOptions(**opts))
    ls = vb.Layer(0.1, 16, engine_options=vb.EngineOptions(**opts))
    ia = vb.TsdfIntegratorFactory.create(kind, vb.TsdfIntegratorConfig(**CFG), la)
    isync = vb.TsdfIntegratorFactory.create(kind, vb.TsdfIntegratorConfig(**CFG), ls)
    offsets = [np.zeros(3), np.array([25.0, 0.0, 0.0]), np.array([0.0, -30.0, 6.0])]
    rooms = scenes.c3_room_sequence(n_scans=21, width=160, height=120)
    scans = [_shifted(s, offsets[i % 3]) for i, s in enumerate(rooms)]
    keep = []
    # one scan at a time first: every scan's counters against the synchronous call's
    for s in scans[:9]:
        isync.integratePointCloud((s[2], s[3]), s[0], s[1])
        keep.append(s)
        ia.integratePointCloudAsync((s[2], s[3]), s[0], s[1])
        la.sync()
        ga, gs = ia.counters(), isync.counters()
        for k in COUNTERS:
            assert ga[k] == gs[k], (k, ga, gs)
    assert _layer_bytes(la) == _layer_bytes(ls)
    # then back to back: both sets in flight
    for s in scans[9:]:
        isync.integratePointCloud((s[2], s[3]), s[0], s[1])
        keep.append(s)
        ia.integratePointCloudAsync((s[2], s[3]), s[0], s[1])
    la.sync()
    assert _layer_bytes(la) == _layer_bytes(ls)
    assert ia.counters()["kernel_launches"] == isync.counters()["kernel_launches"] + 1


def test_pipelined_scans_alternating_between_disjoint_regions(monkeypatch):
    _alternate_between_disjoint_regions(monkeypatch, "merged")


def test_pipelined_simple_scans_alternating_between_disjoint_regions(monkeypatch):
    _alternate_between_disjoint_regions(monkeypatch, "simple")


def _axis_scan():
    """Rays the warp merge does not cover, walked by lane 0 of the trace: points on the three axes through
    the sensor (two zero direction components) and points in the three axis planes through it (one zero
    component), beside ordinary rays that share their blocks."""
    rng = np.random.default_rng(7)
    d = np.linspace(0.6, 3.9, 40, dtype=np.float32)
    pts = []
    for a in range(3):
        for sign in (1.0, -1.0):
            p = np.zeros((d.size, 3), np.float32)
            p[:, a] = sign * d
            pts.append(p)
    for a in range(3):
        p = rng.uniform(-2.5, 2.5, (300, 3)).astype(np.float32)
        p[:, a] = 0.0
        pts.append(p)
    pts.append(rng.uniform(-2.5, 2.5, (2000, 3)).astype(np.float32))
    pts = np.ascontiguousarray(np.concatenate(pts))
    pts = pts[np.linalg.norm(pts, axis=1) > 0.3]
    cols = rng.integers(0, 256, (pts.shape[0], 4), dtype=np.uint8)
    q = np.array([1.0, 0.0, 0.0, 0.0], np.float32)  # identity: the zero components stay exactly zero
    t = np.array([0.0137, -0.0213, 0.0171], np.float32)
    return pts, cols, q, t


def test_sequential_fallback_rays_use_the_scan_table():
    s = _axis_scan()
    layer = vb.Layer(0.1, 16)
    integ = vb.TsdfIntegratorFactory.create("merged", vb.TsdfIntegratorConfig(**CFG), layer)
    ref, port = _reference_map(0.1), _port_map(0.1)
    for scan in (s, _shifted(s, np.array([0.05, 0.0, -0.05]))):
        integ.integratePointCloud((scan[2], scan[3]), scan[0], scan[1])
        ref.integrate(2, scan)
        port.integrate(2, scan)
        gc, oc = integ.counters(), port.counters()
        for k in COUNTERS:
            assert gc[k] == oc[k], (k, gc, oc)
    rep = compare_tsdf(layer, ref)
    print(rep)
    _assert_bit_exact(rep)


def _multi_pass_call(kind, extra):
    """The sensor's block (and its neighbours) receive records in every pass: one local id per block for
    the whole call, so blocks_touched is the call's count, not a sum over passes.  Only the call's last pass
    clears the table: a pass that cleared it early would draw a second id for a block met again."""
    scans = scenes.c3_room_sequence(n_scans=3, width=128, height=96)
    cfg = vb.TsdfIntegratorConfig(**CFG, **extra)
    lp = vb.Layer(0.1, 16, engine_options=vb.EngineOptions(max_updates_per_pass=4096))
    l1 = vb.Layer(0.1, 16)
    ip = vb.TsdfIntegratorFactory.create(kind, cfg, lp)
    i1 = vb.TsdfIntegratorFactory.create(kind, cfg, l1)
    ref, port = _reference_map(0.1, **extra), _port_map(0.1, **extra)
    ref_kind = {"simple": po.SIMPLE, "merged": po.MERGED}[kind]
    for s in scans:
        ip.integratePointCloud((s[2], s[3]), s[0], s[1])
        i1.integratePointCloud((s[2], s[3]), s[0], s[1])
        ref.integrate(ref_kind, s)
        port.integrate(ref_kind, s)
        gp, g1, oc = ip.counters(), i1.counters(), port.counters()
        assert gp["passes"] > 2, gp
        for k in ("rays", "clear_rays", "updates", "blocks_touched", "blocks_allocated"):  # (voxels: summed per pass)
            assert gp[k] == g1[k] == oc[k], (k, gp, g1, oc)
    assert _layer_bytes(lp) == _layer_bytes(l1)
    rep = compare_tsdf(lp, ref)
    print(rep, gp)
    _assert_bit_exact(rep)
    # the table is clean after the passes: a call that fits one pass on the same context still matches
    s = scenes.c3_room_scan(5, width=128, height=96)
    s = (np.ascontiguousarray(s[0][::400]), np.ascontiguousarray(s[1][::400]), s[2], s[3])
    ip.integratePointCloud((s[2], s[3]), s[0], s[1])
    i1.integratePointCloud((s[2], s[3]), s[0], s[1])
    assert ip.counters()["passes"] == 1, ip.counters()
    assert ip.counters()["blocks_touched"] == i1.counters()["blocks_touched"]
    assert _layer_bytes(lp) == _layer_bytes(l1)


def test_multi_pass_call_resolves_each_block_once():
    _multi_pass_call("merged", {})


@pytest.mark.parametrize("kind,extra", [pytest.param("simple", {}, id="simple"),
                                        pytest.param("merged", dict(enable_anti_grazing=1), id="merged_anti_grazing")])
def test_multi_pass_call_of_another_walk_resolves_each_block_once(kind, extra):
    _multi_pass_call(kind, extra)
