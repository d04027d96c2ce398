"""Ownership of the engine's CUDA resources (vbx_engine.h, Holdings).

Without a GPU: only the owner type allocates, creates, frees or destroys device memory, page-locked memory,
streams, events and graphs, so that each resource is released by whoever holds the field it lives in, on every
path.  The page-locked buffers a caller asks for (vbx_host_alloc / vbx_host_free) are the caller's, not the
context's, and are the one exception.

-m gpu: the lifetimes that replace a resource group -- a second vbx_esdf_create, the mesher's and ICP's grow
steps -- and contexts destroyed with asynchronous scans still in flight give the results of fresh contexts."""
import os
import re

import numpy as np
import pytest

import voxblox_b200 as vb
from voxblox_b200 import api, scenes

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "voxblox_b200", "csrc")

RELEASE = ("cudaFree", "cudaFreeHost", "cudaStreamDestroy", "cudaEventDestroy", "cudaGraphExecDestroy",
           "cudaGraphDestroy")
ACQUIRE = ("cudaMalloc", "cudaMallocHost", "cudaHostAlloc", r"cudaStreamCreate\w*", r"cudaEventCreate\w*")
CALLS = re.compile(r"\b(?:%s)\b" % "|".join(RELEASE + ACQUIRE))
OWNER = re.compile(r"\bclass\s+Holdings\b[^;{]*\{")
CALLER_OWNED = re.compile(r"\bint\s+(?:vbx_host_alloc|vbx_host_free)\s*\([^)]*\)\s*\{")


def _code(text):
    """text with comments and the contents of string and character literals blanked (offsets and lines kept)"""
    def blank(m):
        s = m.group(0)
        if s[0] in "\"'":
            return s[0] + re.sub(r"[^\n]", " ", s[1:-1]) + s[-1]
        return re.sub(r"[^\n]", " ", s)
    return re.sub(r"//[^\n]*|/\*.*?\*/|\"(?:\\.|[^\"\\\n])*\"|'(?:\\.|[^'\\\n])*'", blank, text, flags=re.S)


def _block(text, start):
    """[start, end) of the brace block whose '{' is text[start - 1]"""
    depth, i = 1, start
    while depth:
        depth += {"{": 1, "}": -1}.get(text[i], 0)
        i += 1
    return start, i


def test_only_the_owner_type_acquires_or_releases_cuda_resources():
    owner_calls, stray = set(), []
    for f in sorted(os.listdir(CSRC)):
        if not f.endswith((".cu", ".cuh", ".h")):
            continue
        text = _code(open(os.path.join(CSRC, f)).read())
        owners = [_block(text, m.end()) for m in OWNER.finditer(text)]
        allowed = owners + [_block(text, m.end()) for m in CALLER_OWNED.finditer(text)]
        for m in CALLS.finditer(text):
            if any(a <= m.start() < b for a, b in owners):
                owner_calls.add(m.group(0))
            elif not any(a <= m.start() < b for a, b in allowed):
                stray.append(f"{f}:{text.count(chr(10), 0, m.start()) + 1}: {m.group(0)}")
    assert set(RELEASE) <= owner_calls, f"the owner type releases every kind of resource: {sorted(owner_calls)}"
    assert not stray, "acquired or released outside the owner type:\n" + "\n".join(stray)


# ---------------------------------------------------------------------------------------------------- GPU
TSDF_CFG = dict(integrator_threads=1)


def _merged(voxel, vps, trunc, scans, **opts):
    layer = vb.Layer(voxel, vps, engine_options=vb.EngineOptions(**opts) if opts else None)
    integ = vb.TsdfIntegratorFactory.create("merged", vb.TsdfIntegratorConfig(default_truncation_distance=trunc,
                                                                               **TSDF_CFG), layer)
    for s in scans:
        integ.integratePointCloud((s[2], s[3]), s[0], s[1])
    return layer, integ


# The configuration of tests/test_esdf_fixed_point_gpu.py's "min_diff_zero/room_small" cases, whose batch updates
# it holds to the wavefront's fixed point and to the float64 shortest-path reference with no exception.
ESDF_KW = dict(max_distance_m=2.0, default_distance_m=2.0, min_distance_m=0.2, min_diff_m=0.0, multi_queue=1)


def _esdf_batch(recreate):
    """A batch ESDF update of the room's Merged map; with `recreate` on a context whose ESDF was updated after every
    scan (the TSDF's ESDF bits are cleared, the full-Euclidean table allocated) and then created again."""
    from tests.test_esdf_reference_gpu import ROOM_SMALL

    tsdf, integ = _merged(0.1, 16, 0.4, [])
    esdf = vb.Layer(0.1, 16, voxel_type="esdf")
    eint = vb.EsdfIntegrator(vb.EsdfIntegratorConfig(**ESDF_KW), tsdf, esdf)
    for k, s in enumerate(ROOM_SMALL["scans"]()):
        integ.integratePointCloud((s[2], s[3]), s[0], s[1])
        if recreate:
            eint.setFullEuclidean(k == 0)
            eint.updateFromTsdfLayer(True)
    if recreate:
        eint = vb.EsdfIntegrator(vb.EsdfIntegratorConfig(**ESDF_KW), tsdf, esdf)  # vbx_esdf_create again
    eint.updateFromTsdfLayerBatch()
    return esdf.blocks()


@pytest.mark.gpu
def test_esdf_created_again_gives_a_fresh_contexts_batch_update():
    from tests import esdf_fixed_point as fp

    fresh, again = _esdf_batch(False), _esdf_batch(True)
    assert sorted(fresh) == sorted(again)
    for blocks in (fresh, again):
        rep = fp.counts(fp.fixed_point(blocks, 0.1, 16, ESDF_KW, incremental=False, parents=True))
        rep.update({f"dijkstra_{k}": v for k, v in fp.counts(fp.dijkstra_check(blocks, 0.1, 16, ESDF_KW)).items()})
        print(rep)
        assert rep["a"] == 0 and rep["b"] == 0 and rep["c"] in (None, 0), rep
        assert rep["dijkstra_over"] == 0 and rep["dijkstra_under"] == 0, rep
    keys = sorted(fresh)
    f, a = np.stack([fresh[k] for k in keys]), np.stack([again[k] for k in keys])
    assert (f["observed"] == a["observed"]).all() and (f["fixed"] == a["fixed"]).all()
    # the same-sign least fixed point is unique: bit for bit outside the components a sign conflict can reach
    grid, _, tainted = fp.shortest_paths(fresh, 0.1, 16, ESDF_KW)
    _, _, tainted_again = fp.shortest_paths(again, 0.1, 16, ESDF_KW)
    clean = ~(tainted | tainted_again)
    df, da = f["distance"].reshape(-1)[grid.obs_flat], a["distance"].reshape(-1)[grid.obs_flat]
    print("observed", grid.n, "outside sign-conflict components", int(clean.sum()),
          "bit-equal there", int((df[clean] == da[clean]).sum()))
    assert clean.sum() > 0 and (df[clean] == da[clean]).all()


def _mesh(layer):
    mesh_layer = vb.MeshLayer(layer.block_size())
    mesher = vb.MeshIntegrator(vb.MeshIntegratorConfig(), layer, mesh_layer)
    mesher.generateMesh(False, True)
    out = {}
    for i in mesh_layer.getAllAllocatedMeshes():
        m = mesh_layer.getMeshPtrByIndex(i)
        out[tuple(int(v) for v in i)] = (m.vertices.tobytes(), m.normals.tobytes(), m.colors.tobytes())
    return out, mesher.last_blocks, mesher.last_vertices


@pytest.mark.gpu
def test_mesh_after_both_grow_steps_equals_a_fresh_contexts():
    big = [scenes.c3_room_scan(i) for i in range(2)]
    p = big[0][0]
    near = np.nonzero(np.linalg.norm(p - p[len(p) // 2], axis=1) < 0.1)[0]
    small = [(np.ascontiguousarray(p[near]), np.ascontiguousarray(big[0][1][near]), big[0][2], big[0][3])]
    args = (0.02, 8, 0.08)
    layer, integ = _merged(*args, small)
    m_small, nb_small, nv_small = _mesh(layer)
    for s in big:
        integ.integratePointCloud((s[2], s[3]), s[0], s[1])
    m_big, nb_big, nv_big = _mesh(layer)
    layer.removeAllBlocks()
    for s in small:
        integ.integratePointCloud((s[2], s[3]), s[0], s[1])
    m_again, _, _ = _mesh(layer)
    print("small map: blocks", nb_small, "vertices", nv_small, "; larger map: blocks", nb_big, "vertices", nv_big)
    # the first mesh sizes the block group for 256 blocks and the vertex group for 65536 vertices: the larger map
    # outgrows both
    assert 0 < nb_small <= 128 and 0 < nv_small <= 43690 and nb_big > 256 and nv_big > 65536
    assert m_small == _mesh(_merged(*args, small)[0])[0]
    assert m_big == _mesh(_merged(*args, small + big)[0])[0]
    assert m_again == m_small


@pytest.mark.gpu
def test_icp_after_its_grow_step_equals_a_fresh_contexts():
    ss = list(scenes.c3_room_sequence(n_scans=2, width=160, height=120))
    s = ss[1]
    small, large = np.ascontiguousarray(s[0][::40]), s[0]
    assert large.shape[0] > 1024  # (the first call sizes the buffers for max(n, 1024) points)

    def icp(layer, cloud):
        n, (q, t) = vb.ICP(vb.ICPConfig()).runICP(layer, cloud, (s[2], s[3]), seed=9)
        return n, q.tobytes(), t.tobytes()

    layer, _ = _merged(0.1, 16, 0.4, ss[:1])
    grown = [icp(layer, small), icp(layer, large), icp(layer, small)]
    fresh = [icp(_merged(0.1, 16, 0.4, ss[:1])[0], c) for c in (small, large)]
    print("mini batches fused:", [g[0] for g in grown])
    assert grown[1][0] > 0
    assert grown == [fresh[0], fresh[1], fresh[0]]


def _layer_bytes(layer):
    idx = layer.getAllAllocatedBlocks()
    vox, upd = layer.getBlocks(idx)
    return idx.tobytes(), vox.tobytes(), np.asarray(upd).tobytes()


@pytest.mark.gpu
def test_contexts_destroyed_with_scans_in_flight():
    """Each context takes asynchronous scans, uses one of ESDF / mesh / ICP / mirror / device gather, takes more
    asynchronous scans and is destroyed without waiting for them."""
    import torch

    scans = [(np.ascontiguousarray(s[0], np.float32), np.ascontiguousarray(s[1], np.uint8), s[2], s[3])
             for s in scenes.c3_room_sequence(n_scans=4, width=160, height=120)]
    opts = dict(max_blocks=8192, max_points_per_scan=1 << 15, max_updates_per_pass=1 << 22)
    uses = ("esdf", "mesh", "icp", "mirror", "gather")
    first = None
    for k in range(30):
        layer, integ = _merged(0.1, 16, 0.4, [], **opts)
        for s in scans:
            integ.integratePointCloudAsync((s[2], s[3]), s[0], s[1])
        now = _layer_bytes(layer)
        first = first if first is not None else now
        assert now == first, k
        use = uses[k % len(uses)]
        if use == "esdf":
            eint = vb.EsdfIntegrator(vb.EsdfIntegratorConfig(**ESDF_KW), layer, vb.Layer(0.1, 16, voxel_type="esdf"))
            eint.setFullEuclidean(k % 2 == 0)
            eint.updateFromTsdfLayer(True)
        elif use == "mesh":
            assert _mesh(layer)[2] > 0
        elif use == "icp":
            vb.ICP(vb.ICPConfig()).runICP(layer, scans[-1][0], (scans[-1][2], scans[-1][3]), seed=k)
        elif use == "mirror":
            assert layer.stagingBytes() == 0
            idx, _, _ = layer.mirrorUpdated(api.UPDATED_MIRROR, api.UPDATED_MIRROR)
            assert len(idx) > 0 and layer.stagingBytes() > 0
        else:
            n = layer.gatherUpdatedDevice(api.UPDATED_MIRROR)
            d_idx = torch.empty((n, 3), dtype=torch.int32, device="cuda")
            d_vox = torch.empty(n * layer._block_bytes(), dtype=torch.uint8, device="cuda")
            assert n > 0 and layer.gatherUpdatedDevice(api.UPDATED_MIRROR, api.UPDATED_MIRROR, False, d_idx, d_vox) == n
        for s in scans:
            integ.integratePointCloudAsync((s[2], s[3]), s[0], s[1])
        layer._ctx.close()  # vbx_destroy with the scans just submitted in flight
