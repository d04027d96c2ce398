"""The full-Euclidean ESDF checker (tests/esdf_fe_check.py) on its own, without a GPU: the device's word order on
hand-made pairs; the restatement's full-Euclidean layers of the wall and room_small, batch and incremental, with
what the reference's own rules break printed; and single-voxel mutations of a clean layer, each named exactly at
the mutated voxel."""
import numpy as np
import pytest

from oracle import pyoracle as po
from tests import esdf_fe_check as fc
from tests.test_esdf_gpu import _wall_scans
from tests import test_esdf_reference_gpu as te

F32 = np.float32
P0 = np.zeros(3, np.int32)


def _w(d, p=(0, 0, 0)):
    return int(fc.word(np.array([d], F32), np.array([p], np.int32))[0])


def test_word_order():
    """Words order as the device's signed 64-bit atomicMin does: -0.0 below every inside value, +0.0 above them,
    inside values nearer zero smaller, outside values in float order, equal distances by parent code (x low)."""
    assert _w(-0.0) < _w(-1e-30) < _w(-0.1) < _w(-0.2) < _w(-2.0)
    assert _w(-2.0) < _w(0.0) < _w(1e-30) < _w(0.1) < _w(0.2)
    assert _w(-0.0, (511, 511, 511)) < _w(-0.1, (-512, -512, -512))
    assert _w(0.3, (-1, 0, 0)) < _w(0.3, (0, 0, 0)) < _w(0.3, (1, 0, 0)) < _w(0.3, (-512, 1, 0)) < _w(0.3, (0, 0, 1))
    assert _w(-0.3, (0, -1, 0)) < _w(-0.3, (5, 0, 0)) < _w(-0.3, (-5, 0, 1))  # y above x, z above y
    # a component outside [-512, 511] does not survive the 10-bit code
    p = np.array([[511, -512, 0], [512, 0, 0], [0, -513, 0]], np.int32)
    assert (fc.parent_decode(fc.parent_code(p)) == p).all(1).tolist() == [True, False, False]
    assert fc.parent_ok(p).tolist() == [True, False, False]


def _restated(scene, incremental):
    """The restatement's full-Euclidean layers: (checked (incremental, before, after) updates, voxel, vps, ekw)."""
    if scene == "wall":
        voxel, trunc, max_d, scans = 0.1, 0.4, 4.0, _wall_scans()
    else:
        voxel, trunc, max_d, scans = 0.1, 0.4, 2.0, te.ROOM_SMALL["scans"]()
    ekw = dict(max_distance_m=max_d, default_distance_m=max_d, min_distance_m=trunc / 2, min_diff_m=0.0, multi_queue=1,
               full_euclidean_distance=1)
    omap = po.OracleMap(po.OracleLib("port"), po.TsdfConfig(default_truncation_distance=trunc), voxel, 16)
    omap.esdf_create(po.EsdfConfig(**ekw))
    out = []
    for s in scans:
        omap.integrate(2, s)
        if incremental:
            before = omap.blocks(1)
            omap.esdf_update(batch=False)
            out.append((True, before, omap.blocks(1)))
    if not incremental:
        omap.esdf_update(batch=True)
        out.append((False, None, omap.blocks(1)))
    return out, voxel, 16, ekw


# measured on the restatement (held digest for digest to the reference's EsdfIntegrator elsewhere): what its own
# pop order leaves behind, summed over the checked updates.  Its batch layers break (a) only through the mixed-sign
# rule, and (t) where a chain crossed the surface twice; its incremental updates leave children of raised voxels
# rooted through them (s_parent_raised) on room_small
RESTATED = {
    ("wall", False): dict(a=0, r_other=0, t=0),
    ("room_small", False): dict(a=12, a_mixed=12, r_other=0, r_fixed_other=1742, t=1822),
    ("wall", True): dict(a=12, a_stale_source=12, r_other=0, t=4364, s_parent_raised=0),
    ("room_small", True): dict(a=58, a_other=1, r_other=414, t=4972, s_parent_raised=379),
}


@pytest.mark.parametrize("scene,incremental", list(RESTATED))
def test_restated_layers(scene, incremental):
    steps, voxel, vps, ekw = _restated(scene, incremental)
    total = {}
    for inc, before, after in steps:
        rep = fc.counts(fc.fe_check(after, voxel, vps, ekw, incremental=inc, before=before))
        for k, v in rep.items():
            if isinstance(v, int):
                total[k] = total.get(k, 0) + v
    if not incremental:
        e = fc.euclidean(steps[-1][2], voxel, vps, ekw)
        print(scene, "EDT", {k: v for k, v in e.items() if k not in ("edt", "grid", "under")})
        assert len(e["under"]) <= total["t"]
    print(scene, "incremental" if incremental else "batch", "reference breaks:", total)
    assert total["range"] == 0
    for k, v in RESTATED[(scene, incremental)].items():
        if v is not None:
            assert total[k] == v, (k, total)


# ------------------------------------------------------------------ mutations of a clean layer
VPS = 4


@pytest.fixture(scope="module")
def clean():
    """The restatement's batch layer of two fixed voxels in a cube of free voxels: nothing fires, every root is a
    fixed voxel of the same sign, every voxel is on the telescoping identity and on the EDT."""
    g, d = fc.synthetic("two_points")
    blocks = fc.oracle_layer(po.OracleLib("port"), g, d, VPS, fc.SYN_EKW).blocks(1)
    rep = fc.fe_check(blocks, fc.SYN_VOXEL, VPS, fc.SYN_EKW)
    c = fc.counts(rep)
    assert c["a"] == c["range"] == c["t"] == c["r_other"] == c["r_seeded"] == c["r_fixed_other"] == 0, c
    assert c["r_fixed_same"] == c["reached"] == len(g) - 2
    return blocks, rep


@pytest.fixture(scope="module")
def hairpin():
    """The restatement's batch layer of the hairpin path: the way back past the turn is unreached."""
    g, d = fc.synthetic("hairpin")
    blocks = fc.oracle_layer(po.OracleLib("port"), g, d, VPS, fc.SYN_EKW).blocks(1)
    rep = fc.fe_check(blocks, fc.SYN_VOXEL, VPS, fc.SYN_EKW)
    c = fc.counts(rep)
    assert c["a"] == c["t"] == c["r_other"] == c["r_seeded"] == 0 and c["r_fixed_same"] == c["reached"] == 9, c
    return blocks, rep


def _slot(blocks, g):
    b = tuple(int(c) // VPS for c in g)
    x, y, z = (int(c) - VPS * bc for c, bc in zip(g, b))
    return blocks[b], x + VPS * (y + VPS * z)


def _neighbourhood(g):
    return {tuple(int(c) for c in np.add(g, o)) for o in fc.K_OFF} | {tuple(g)}


PER_VOXEL = ("range", "r_fixed_other", "r_seeded", "r_unit", "r_other", "t")


def _mutate(blocks, rep, mutation):
    """(mutated layer, voxel, lists that must name it)."""
    m = {k: v.copy() for k, v in blocks.items()}
    grid = fc.Grid(blocks, VPS)
    names = [tuple(int(c) for c in x) for x in grid.gidx]
    pos = {x: i for i, x in enumerate(names)}
    n2 = (grid.parent.astype(np.int64) ** 2).sum(1)
    reached = [x for x in fc.as_set(rep["r_fixed_same"])]
    reached.sort()
    if mutation == "value_beyond_tolerance":
        g = max(reached, key=lambda x: n2[pos[x]])
        vox, lin = _slot(m, g)
        tol = fc.tolerance(n2[pos[g]:pos[g] + 1], fc.SYN_VOXEL, fc.SYN_EKW)[0]
        vox["distance"][lin] = F32(vox["distance"][lin] + 2 * tol + 1e-6)
        return m, g, ("t", "a")
    if mutation == "parent_plus_one":
        g = next(x for x in reached if n2[pos[x]] >= 9)
        vox, lin = _slot(m, g)
        vox["parent"][lin][0] += 1
        return m, g, ("r_other",)
    if mutation == "parent_tie_smaller_code":
        # the same |parent| (the telescoped distance ties) and a smaller parent code: a permutation of the components
        for g in reached:
            p = grid.parent[pos[g]]
            for q in (p[[1, 0, 2]], p[[0, 2, 1]], p[[2, 1, 0]], p[[1, 2, 0]], p[[2, 0, 1]]):
                j = grid.lookup(np.array([np.add(g, q)]))[0]
                if (q != p).any() and fc.parent_code(q) < fc.parent_code(p) and (j < 0 or not grid.fixed[j]):
                    vox, lin = _slot(m, g)
                    vox["parent"][lin] = q
                    return m, g, ("r_other",)
        raise AssertionError("no voxel whose parent has a smaller permutation")
    if mutation == "negative_step_lower":
        # (on the hairpin layer) the first voxel of the way back is unreached: its only source offers a candidate
        # with a negative step (what the wavefront would write without the dist < 0 skip, cc:423-425); written as
        # the value alone, the voxel is reached with parent 0, so its root is itself and not fixed
        g = (fc.HAIRPIN_L - 1, 3, 0)
        s = pos[(fc.HAIRPIN_L, 3, 0)]
        assert grid.d[pos[g]] == F32(fc.SYN_EKW["default_distance_m"])
        _, step = fc.fe_step(fc.SYN_VOXEL, grid.parent[s:s + 1], 0)     # towards -x
        assert step[0] < 0
        vox, lin = _slot(m, g)
        vox["distance"][lin] = F32(grid.d[s] + step[0])
        return m, g, ("r_seeded",)
    if mutation == "root_not_fixed":
        g = next(x for x in reached if n2[pos[x]] >= 4)
        root = tuple(int(c) for c in np.add(g, grid.parent[pos[g]]))
        vox, lin = _slot(m, root)
        vox["fixed"][lin] = 0
        # every voxel rooted there loses its fixed root: the mutated voxel is the root, which is now reached
        return m, root, None
    if mutation == "parent_code_512":
        g = next(x for x in reached if n2[pos[x]] >= 4)
        vox, lin = _slot(m, g)
        vox["parent"][lin][0] = 512
        return m, g, ("range", "r_other")
    raise KeyError(mutation)


MUTATIONS = ["value_beyond_tolerance", "parent_plus_one", "parent_tie_smaller_code", "negative_step_lower",
             "root_not_fixed", "parent_code_512"]


@pytest.mark.parametrize("mutation", MUTATIONS)
def test_mutation_named(request, mutation):
    """Each mutation is named at the mutated voxel by the lists it must be in, and by no other per-voxel list
    anywhere else; (a) names, if anything, only the voxel and its neighbours (a changed source)."""
    blocks, base = request.getfixturevalue("hairpin" if mutation == "negative_step_lower" else "clean")
    m, g, want = _mutate(blocks, base, mutation)
    rep = fc.fe_check(m, fc.SYN_VOXEL, VPS, fc.SYN_EKW)
    print(mutation, g, fc.counts(rep))
    if mutation == "root_not_fixed":
        # the root is reached now (observed, not fixed, not at default): its own root is itself with parent 0, and
        # every voxel rooted at it is rooted at a non-fixed voxel with parent 0
        rooted_there = {x for x in fc.as_set(base["r_fixed_same"])
                        if tuple(np.add(x, fc.Grid(blocks, VPS).parent[fc.Grid(blocks, VPS).lookup(np.array([x]))[0]]))
                        == g}
        assert fc.as_set(rep["r_seeded"]) == rooted_there | {g}
        assert all(len(rep[k]) == 0 for k in PER_VOXEL if k != "r_seeded"), fc.counts(rep)
        return
    for k in PER_VOXEL:
        added = fc.as_set(rep[k]) - fc.as_set(base[k])
        assert added == ({g} if k in want else set()), (k, added)
        assert fc.as_set(base[k]) - fc.as_set(rep[k]) == set(), k
    a = fc.as_set(rep["a"])
    assert a <= _neighbourhood(g), a
    if "a" in want:
        assert g in a
