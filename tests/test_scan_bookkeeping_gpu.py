"""-m gpu: what a call reports about itself -- the stages it timed, the kernels it launched and the counters of
its last scan.  A synchronous call counts each kernel where it is launched; a pipelined scan's count is the
number of kernel nodes in its graph, which is the synchronous call's kernels plus k_back_begin.  A synchronous
call and a collected asynchronous scan fill their counters through the same code."""
import numpy as np
import pytest

import voxblox_b200 as vb
from voxblox_b200 import scenes

pytestmark = pytest.mark.gpu

CFG = dict(default_truncation_distance=0.4, integrator_threads=1)
OPTS = dict(max_updates_per_pass=1 << 22)  # no scan here needs a second pass (or an asynchronous redo)

# stages a synchronous call times with stage profiling on
STAGES = {
    "simple": {"ray_count", "scan", "ray_emit", "assign", "update_sort", "apply"},
    "merged": {"point_keys", "point_sort", "bundle_order", "bundle_merge", "ray_count", "scan", "ray_emit",
               "assign", "update_sort", "apply"},
}
# kernels a synchronous call launches; a pipelined scan adds k_back_begin
LAUNCHES = {"simple": 7, "merged": 14}


def _scans(n):
    return scenes.c3_room_sequence(n_scans=n, width=128, height=96)


def _called(layer):
    return {k for k, (_, calls) in layer.stageMs().items() if calls}


@pytest.mark.parametrize("kind", ["simple", "merged"])
def test_stages_and_launches_of_a_scan(kind):
    layer = vb.Layer(0.1, 16, engine_options=vb.EngineOptions(**OPTS))
    integ = vb.TsdfIntegratorFactory.create(kind, vb.TsdfIntegratorConfig(**CFG), layer)
    layer.setStageProfiling(True)
    scans = _scans(4)
    for s in scans[:2]:
        integ.integratePointCloud((s[2], s[3]), s[0], s[1])
        assert integ.counters()["kernel_launches"] == LAUNCHES[kind], integ.counters()
    assert _called(layer) == STAGES[kind]
    assert all(layer.stageMs()[k][1] == 2 for k in STAGES[kind])
    for s in scans[2:]:
        integ.integratePointCloudAsync((s[2], s[3]), s[0], s[1])
        layer.sync()
        assert integ.counters()["kernel_launches"] == LAUNCHES[kind] + 1, integ.counters()
    # the graphs record no stage events
    assert _called(layer) == STAGES[kind]
    assert all(layer.stageMs()[k][1] == 2 for k in STAGES[kind])


def test_stages_and_launches_of_an_esdf_update():
    layer = vb.Layer(0.1, 16)
    integ = vb.TsdfIntegratorFactory.create("merged", vb.TsdfIntegratorConfig(**CFG), layer)
    for s in _scans(2):
        integ.integratePointCloud((s[2], s[3]), s[0], s[1])
    esdf = vb.Layer(0.1, 16, voxel_type="esdf")
    eint = vb.EsdfIntegrator(vb.EsdfIntegratorConfig(max_distance_m=2.0, default_distance_m=2.0), layer, esdf)
    layer.setStageProfiling(True)
    eint.updateFromTsdfLayerBatch()
    assert _called(layer) == {"esdf_propagate", "esdf_raise", "esdf_lower"}
    # block list, propagate, raise, lower, parents
    assert eint.counters()["kernel_launches"] == 5, eint.counters()


@pytest.mark.parametrize("kind", ["simple", "merged"])
def test_asynchronous_and_synchronous_scans_report_the_same_counters(kind):
    la = vb.Layer(0.1, 16, engine_options=vb.EngineOptions(**OPTS))
    ls = vb.Layer(0.1, 16, engine_options=vb.EngineOptions(**OPTS))
    ia = vb.TsdfIntegratorFactory.create(kind, vb.TsdfIntegratorConfig(**CFG), la)
    isync = vb.TsdfIntegratorFactory.create(kind, vb.TsdfIntegratorConfig(**CFG), ls)
    keep = []
    for s in _scans(9):
        isync.integratePointCloud((s[2], s[3]), s[0], s[1])
        p, c = np.ascontiguousarray(s[0]), np.ascontiguousarray(s[1])
        keep.append((p, c))
        ia.integratePointCloudAsync((s[2], s[3]), p, c)
    la.sync()
    ga, gs = ia.counters(), isync.counters()
    assert ga["async_redone_total"] == 0, ga
    if kind == "merged":
        assert gs["bundle_key_bits"] > 0, gs
    for k in gs:
        if k.endswith("_total"):
            continue
        want = gs[k] + 1 if k == "kernel_launches" else gs[k]
        assert ga[k] == want, (k, ga, gs)
