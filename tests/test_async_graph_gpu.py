"""-m gpu: pipelined submission runs each scan as one launch of a CUDA graph captured once per (hand-off set,
front lane, variant).  Everything that changes from scan to scan -- point count, pose, cloud pointers, the
block-count word, the record sort's grid, k_bundle_order's shared memory and form -- must reach the graph,
and the events between graphs must keep the map-touching stages in submission order.  Each case compares
the asynchronously built map with the synchronous calls' bit for bit (distance, weight, colour, updated
bits, block set)."""
import numpy as np
import pytest

import voxblox_b200 as vb
from voxblox_b200 import scenes

pytestmark = pytest.mark.gpu

CFG = dict(default_truncation_distance=0.4, integrator_threads=1)


def _layer_bytes(layer):
    idx = layer.getAllAllocatedBlocks()
    vox, upd = layer.getBlocks(idx)
    return idx.tobytes(), vox.tobytes(), np.asarray(upd).tobytes()


def _scatter_scan(pose_scan, n=40000, seed=1):
    """points scattered through the room: nearly every point is its own bundle (k_bundle_order's
    cooperative form, > 18 k bundles)"""
    rng = np.random.default_rng(seed)
    pts = rng.uniform(-3.5, 3.5, (n, 3)).astype(np.float32)
    col = rng.integers(0, 256, (n, 4), dtype=np.uint8)
    return pts, col, pose_scan[2], pose_scan[3]


def _thin(s, keep, seed):
    """a random subset of the scan's points (point counts that vary from scan to scan)"""
    rng = np.random.default_rng(seed)
    sel = np.sort(rng.choice(s[0].shape[0], size=keep, replace=False))
    return np.ascontiguousarray(s[0][sel]), np.ascontiguousarray(s[1][sel]), s[2], s[3]


class Pair:
    """the same scans into an asynchronously and a synchronously fed map"""

    def __init__(self, kind="merged", **opts):
        o = dict(max_updates_per_pass=1 << 22)
        o.update(opts)
        self.la = vb.Layer(0.1, 16, engine_options=vb.EngineOptions(**o))
        self.ls = vb.Layer(0.1, 16, engine_options=vb.EngineOptions(**o))
        self.ia = vb.TsdfIntegratorFactory.create(kind, vb.TsdfIntegratorConfig(**CFG), self.la)
        self.isync = vb.TsdfIntegratorFactory.create(kind, vb.TsdfIntegratorConfig(**CFG), self.ls)
        self.keep = []

    def add(self, s, host="pageable"):
        self.isync.integratePointCloud((s[2], s[3]), s[0], s[1])
        if host == "pinned":
            p, c = self.la.hostBuffer(s[0].shape, np.float32), self.la.hostBuffer(s[1].shape, np.uint8)
            p[...] = s[0]
            c[...] = s[1]
        else:
            p, c = np.ascontiguousarray(s[0]), np.ascontiguousarray(s[1])
        self.keep.append((p, c))
        self.ia.integratePointCloudAsync((s[2], s[3]), p, c)

    def check(self):
        self.la.sync()
        assert _layer_bytes(self.la) == _layer_bytes(self.ls)
        # a pipelined scan runs the synchronous call's kernels plus k_back_begin (kernel nodes executed)
        assert self.ia.counters()["kernel_launches"] == self.isync.counters()["kernel_launches"] + 1


@pytest.mark.parametrize("kind", ["simple", "merged"])
def test_point_counts_that_vary_widely(kind):
    p = Pair(kind)
    scans = scenes.c3_room_sequence(n_scans=12, width=160, height=120)
    full = scans[0][0].shape[0]
    for i, s in enumerate(scans):
        keep = [full, 37, full // 2, 5000, 1, full // 7][i % 6]
        p.add(_thin(s, min(keep, s[0].shape[0]), i), host="pinned" if i % 2 else "pageable")
    p.check()


def test_bundle_count_jumps_between_the_order_forms():
    """k_bundle_order: the cooperative form (no hint yet, and after a scan of ~40 k bundles) and the
    one-block form with a shared-memory request that follows the bundle count of recent scans"""
    p = Pair("merged", max_updates_per_pass=1 << 23)
    rooms = scenes.c3_room_sequence(n_scans=8, width=160, height=120)
    big = _scatter_scan(rooms[0])
    p.add(rooms[0])                    # cooperative: nothing is known about the bundle count yet
    p.add(rooms[1])
    p.la.sync()                        # the hint becomes the room scans' count: one block, small request
    p.add(rooms[2])
    p.add(_thin(rooms[3], 300, 3))
    p.add(big)
    p.la.sync()                        # the hint is now ~40 k bundles: the cooperative form
    p.add(rooms[4])
    p.add(big)
    p.la.sync()
    p.add(_thin(rooms[5], 2000, 5))    # and back to the one-block form
    p.add(rooms[6])
    p.check()


@pytest.mark.parametrize("sets,lanes", [(7, 3), (3, 7), (5, 5), (2, 1)])
def test_odd_set_and_lane_counts(monkeypatch, sets, lanes):
    """the block-count ping-pong word alternates per scan, which an odd set count does not follow"""
    monkeypatch.setenv("VBX_ASYNC_SETS", str(sets))
    monkeypatch.setenv("VBX_ASYNC_LANES", str(lanes))
    p = Pair("merged")
    for s in scenes.c3_room_sequence(n_scans=23, width=128, height=96):
        p.add(s)
    p.check()


def test_more_sets_than_scans(monkeypatch):
    monkeypatch.setenv("VBX_ASYNC_SETS", "16")
    p = Pair("merged")
    for s in scenes.c3_room_sequence(n_scans=5, width=128, height=96):
        p.add(s)
    p.check()
    for s in scenes.c3_room_sequence(n_scans=3, width=128, height=96, start=5):
        p.add(s)
    p.check()


def test_synchronous_calls_and_block_edits_between_batches():
    p = Pair("merged")
    scans = scenes.c3_room_sequence(n_scans=14, width=128, height=96)
    for s in scans[:4]:
        p.add(s)
    # a synchronous call queues behind the asynchronous ones
    for layer, integ in ((p.la, p.ia), (p.ls, p.isync)):
        integ.integratePointCloud((scans[4][2], scans[4][3]), scans[4][0], scans[4][1])
    for s in scans[5:8]:
        p.add(s, host="pinned")
    p.la.sync()
    # block removals and uploads change the block count the next scan's k_assign starts from
    idx = p.ls.getAllAllocatedBlocks()
    assert (idx == p.la.getAllAllocatedBlocks()).all()
    gone = idx[::5]
    vox, upd = p.ls.getBlocks(idx[1:3])
    moved = idx[1:3] + np.array([0, 0, 40], np.int32)
    for layer in (p.la, p.ls):
        layer.removeBlocks(gone)
        layer.insertBlocks(moved, vox, upd)
    for s in scans[8:12]:
        p.add(s)
    p.la.sync()
    p.la.sync()
    for s in scans[12:]:
        p.add(s)
    p.check()


def test_over_capacity_scan_in_the_middle_of_the_queue_is_redone():
    """the scattered scan has more update records than one pass holds: it and the scans queued behind it
    skip their back halves and are redone synchronously, in submission order"""
    p = Pair("merged", max_updates_per_pass=1 << 20)
    rooms = scenes.c3_room_sequence(n_scans=9, width=128, height=96)
    for i, s in enumerate(rooms):
        p.add(s)
        if i == 3:
            p.add(_scatter_scan(s))
    p.la.sync()
    assert p.ia.counters()["async_redone_total"] >= 1
    assert p.isync.counters()["passes"] > 0
    assert _layer_bytes(p.la) == _layer_bytes(p.ls)


@pytest.mark.parametrize("host", ["pageable", "pinned", "device"])
def test_host_and_device_clouds(host):
    torch = pytest.importorskip("torch")
    p = Pair("merged")
    scans = scenes.c3_room_sequence(n_scans=9, width=160, height=120)
    dev = []
    for i, s in enumerate(scans):
        if host != "device":
            p.add(s, host=host)
            continue
        p.isync.integratePointCloud((s[2], s[3]), s[0], s[1])
        x, c = torch.from_numpy(s[0]).cuda(), torch.from_numpy(s[1]).cuda()
        dev.append((x, c))
        torch.cuda.synchronize()
        p.ia.integratePointCloudAsync((s[2], s[3]), x.data_ptr(), c.data_ptr(), int(s[0].shape[0]))
    p.check()
