"""The ESDF fixed-point checker (tests/esdf_fixed_point.py) on its own, without a GPU: on the restatement's batch
ESDF of the wall scene it reports what it must, and on single-voxel mutations of that layer it names exactly
the voxel that was changed."""
import numpy as np
import pytest

from oracle import pyoracle as po
from tests import esdf_fixed_point as fp
from tests.test_esdf_gpu import EKW, _wall_scans

VOXEL, VPS = 0.1, 16


@pytest.fixture(scope="module")
def wall():
    omap = po.OracleMap(po.OracleLib("port"), po.TsdfConfig(default_truncation_distance=0.4), VOXEL, VPS)
    omap.esdf_create(po.EsdfConfig(**EKW))
    for s in _wall_scans():
        omap.integrate(2, s)
    omap.esdf_update(batch=True)
    blocks = omap.blocks(1)
    return blocks, fp.fixed_point(blocks, VOXEL, VPS, EKW), fp.dijkstra_check(blocks, VOXEL, VPS, EKW)


def _copy(blocks):
    return {k: v.copy() for k, v in blocks.items()}


def _at(blocks, g):
    """(block, linear index) of global voxel index g."""
    b = tuple(int(c) // VPS for c in g)
    x, y, z = (int(c) - VPS * bc for c, bc in zip(g, b))
    return blocks[b], x + VPS * (y + VPS * z)


def _value(blocks, g):
    vox = blocks.get(tuple(int(c) // VPS for c in g))
    if vox is None:
        return None
    v, lin = _at(blocks, g)
    return v[lin] if v[lin]["observed"] else None


def _leaves(blocks):
    """Reached, non-fixed voxels no observed neighbour lies farther from the surface than: nothing derives its
    value from theirs, so changing one changes no other voxel's status."""
    dflt = np.float32(EKW["default_distance_m"])
    out = []
    for b, vox in sorted(blocks.items()):
        for lin in np.nonzero((vox["observed"] != 0) & (vox["fixed"] == 0))[0]:
            d = vox["distance"][lin]
            if abs(d) == dflt:
                continue
            g = np.array(b) * VPS + [lin % VPS, (lin // VPS) % VPS, lin // VPS ** 2]
            nbrs = [_value(blocks, g + o) for o in fp.K_OFF]
            if all(n is None or (abs(n["distance"]) <= abs(d) and (n["distance"] > 0) == (d > 0)) for n in nbrs):
                out.append(tuple(int(c) for c in g))
            if len(out) == 16:
                return out
    return out


def _reproduced(blocks, g, value):
    """Does a neighbour of voxel g reproduce `value` through one same-sign step (plain loop)?"""
    for k, o in enumerate(fp.K_OFF):
        n = _value(blocks, np.array(g) + o)
        if n is None or abs(n["distance"]) >= np.float32(EKW["max_distance_m"]) or (n["distance"] > 0) != (value > 0):
            continue
        step = np.float32(np.float32([1.0, np.sqrt(2.0), np.sqrt(3.0)][0 if k < 6 else (1 if k < 18 else 2)]) * np.float32(VOXEL))
        if np.float32(abs(n["distance"]) + step) == abs(value):
            return True
    return False


def _new(rep, base, what):
    return fp.as_set(rep[what]) - fp.as_set(base[what]), fp.as_set(base[what]) - fp.as_set(rep[what])


def test_wall_batch_reports(wall):
    """The restatement's batch update of the wall: nothing can fire, every value is justified, the float64
    reference agrees on every voxel; the reference's own parents are its last writers, not the first justifier in
    table order, at 17 voxels (ties)."""
    blocks, rep, dj = wall
    print(fp.counts(rep), fp.counts(dj))
    assert (rep["observed"], rep["reached"]) == (20755, 15423)
    assert len(rep["a"]) == 0 and len(rep["b"]) == 0 and len(rep["c"]) == 17
    assert dj["compared"] == dj["clean"] == 15423
    assert len(dj["over"]) == 0 and len(dj["under"]) == 0


@pytest.mark.parametrize("mutation", ["plus_ulp", "minus_ulp", "default", "half_step_low", "parent"])
def test_mutation_named(wall, mutation):
    blocks, base, base_dj = wall
    leaves = _leaves(blocks)
    assert leaves, "the wall scene has voxels nothing derives from"
    m = _copy(blocks)
    if mutation in ("plus_ulp", "minus_ulp"):
        # one ulp further from / nearer to the surface, at a leaf where no neighbour happens to reproduce that
        def moved(g):
            d = _value(blocks, np.array(g))["distance"]
            return np.nextafter(d, np.float32(np.sign(d) * (np.inf if mutation == "plus_ulp" else 0)))
        g = next(x for x in leaves if not _reproduced(blocks, x, moved(x)))
        vox, lin = _at(m, g)
        vox["distance"][lin] = moved(g)
    else:
        g = leaves[0]
        vox, lin = _at(m, g)
        d = vox["distance"][lin]
    if mutation == "default":
        vox["distance"][lin] = np.sign(d) * np.float32(EKW["default_distance_m"])
    elif mutation == "half_step_low":
        vox["distance"][lin] = d - np.sign(d) * np.float32(VOXEL / 2)
    elif mutation == "parent":  # a voxel that is its children's source: flip its parent
        rep_c = fp.as_set(base["c"])
        cand = [tuple(int(c) for c in x) for x in fp.Grid(blocks, VPS).gidx]
        g = next(x for x in cand if x not in rep_c and x not in leaves and _value(blocks, np.array(x)) is not None
                 and not _value(blocks, np.array(x))["fixed"] and (_value(blocks, np.array(x))["parent"] != 0).any())
        vox, lin = _at(m, g)
        vox["parent"][lin] = -vox["parent"][lin]
    rep = fp.fixed_point(m, VOXEL, VPS, EKW)
    dj = fp.dijkstra_check(m, VOXEL, VPS, EKW)
    want = {"plus_ulp": ("a", "b"), "minus_ulp": ("b",), "default": ("a", "over"), "half_step_low": ("b", "under"),
            "parent": ("c",)}[mutation]
    for what in ("a", "b", "c", "over", "under"):
        r, bs = (dj, base_dj) if what in ("over", "under") else (rep, base)
        added, gone = _new(r, bs, what)
        print(mutation, g, what, sorted(added), sorted(gone))
        assert gone == set(), (what, gone)
        assert added == ({g} if what in want else set()), (what, added)


def test_removed_block_named(wall):
    """Removing an ESDF block removes its voxels as neighbours: the checker names exactly the voxels next to it
    whose every justifier lay inside it (b), and those whose first justifier in table order did (c)."""
    blocks, base, _ = wall
    # the block with the most reached voxels, among blocks with a neighbour block on every face
    def reached(v):
        return int(((v["observed"] != 0) & (v["fixed"] == 0) & (np.abs(v["distance"]) < EKW["default_distance_m"])).sum())
    inner = [k for k in blocks if all(tuple(np.add(k, o)) in blocks for o in fp.K_OFF[:6])]
    gone_block = max(inner, key=lambda k: reached(blocks[k]))
    m = _copy(blocks)
    del m[gone_block]
    rep = fp.fixed_point(m, VOXEL, VPS, EKW)
    # plain loops over the voxels next to the removed block: which justifiers lay inside it
    d1, d2, d3 = (np.float32(np.float32(s) * np.float32(VOXEL)) for s in (1.0, np.sqrt(2.0), np.sqrt(3.0)))
    lo, hi = np.array(gone_block) * VPS - 1, np.array(gone_block) * VPS + VPS
    want_b, want_c = set(), set()
    for x in range(lo[0], hi[0] + 1):
        for y in range(lo[1], hi[1] + 1):
            for z in range(lo[2], hi[2] + 1):
                g = np.array([x, y, z])
                if (lo < g).all() and (g < hi).all():
                    continue
                v = _value(blocks, g)
                if v is None or v["fixed"] or abs(v["distance"]) == np.float32(EKW["default_distance_m"]):
                    continue
                just = []
                for k, o in enumerate(fp.K_OFF):
                    n = _value(blocks, g + o)
                    if n is None or abs(n["distance"]) >= np.float32(EKW["max_distance_m"]):
                        continue
                    step = d1 if k < 6 else (d2 if k < 18 else d3)
                    if (n["distance"] > 0) == (v["distance"] > 0) and np.float32(abs(n["distance"]) + step) == abs(v["distance"]):
                        just.append(k)
                inside = [tuple(g + fp.K_OFF[k]) for k in just]
                kept = [k for k, t in zip(just, inside) if not all(lo < t) or not all(np.array(t) < hi)]
                if just and not kept:
                    want_b.add((x, y, z))
                elif kept and kept[0] != just[0] and (v["parent"] != fp.K_OFF[kept[0]]).any():
                    want_c.add((x, y, z))
    print("removed", gone_block, "b", len(want_b), "c", len(want_c))
    assert want_b, "the removed block justifies voxels next to it"
    assert fp.as_set(rep["b"]) == want_b
    assert len(rep["a"]) == 0
    assert fp.as_set(rep["c"]) - fp.as_set(base["c"]) == want_c


def _one_block(cells):
    """A one-block layer (voxels per side 4) holding `cells`: {(x, y, z): (distance, fixed, parent)}."""
    vox = np.zeros(64, po.ESDF_DTYPE)
    for (x, y, z), (d, fixed, parent) in cells.items():
        lin = x + 4 * (y + 4 * z)
        vox[lin]["observed"] = 1
        vox[lin]["distance"] = d
        vox[lin]["fixed"] = fixed
        vox[lin]["parent"] = parent
    return {(0, 0, 0): vox}


def test_mixed_sign_rule():
    """A fixed voxel just outside the surface next to an unreached inside voxel: the mixed-sign rule of
    k_esdf_lower lowers the inside voxel to -step (a) until it holds that value, which then justifies it (b)
    with its parent pointing at the outside voxel (c)."""
    ekw = dict(max_distance_m=2.0, default_distance_m=2.0, min_diff_m=0.0)
    step = np.float32(np.float32(1.0) * np.float32(VOXEL))
    src = ((1, 1, 1), (np.float32(0.05), 1, (0, 0, 0)))
    rep = fp.fixed_point(_one_block(dict([src, ((2, 1, 1), (np.float32(-2.0), 0, (0, 0, 0)))])), VOXEL, 4, ekw)
    assert fp.as_set(rep["a"]) == {(2, 1, 1)} and len(rep["b"]) == 0
    ok = _one_block(dict([src, ((2, 1, 1), (-step, 0, (-1, 0, 0)))]))
    rep = fp.fixed_point(ok, VOXEL, 4, ekw)
    assert len(rep["a"]) == 0 and len(rep["b"]) == 0 and len(rep["c"]) == 0
    bad = _one_block(dict([src, ((2, 1, 1), (-step, 0, (1, 0, 0)))]))
    assert fp.as_set(fp.fixed_point(bad, VOXEL, 4, ekw)["c"]) == {(2, 1, 1)}
    wrong = _one_block(dict([src, ((2, 1, 1), (np.float32(-0.15), 0, (-1, 0, 0)))]))
    rep = fp.fixed_point(wrong, VOXEL, 4, ekw)
    assert fp.as_set(rep["a"]) == {(2, 1, 1)} and fp.as_set(rep["b"]) == {(2, 1, 1)}


def test_incremental_classes():
    """An unscaled seed value next to a source that could lower it is class a_seed; a value no neighbour
    justifies any more that the update left as it was is b_stale; the same value changed by the update is
    b_other."""
    ekw = dict(max_distance_m=2.0, default_distance_m=2.0, min_diff_m=0.0)
    fixed = ((1, 1, 1), (np.float32(0.05), 1, (0, 0, 0)))
    seeded = ((2, 1, 1), (np.float32(np.float32(0.05) + np.float32(1.0)), 0, (0, 0, 0)))
    rep = fp.fixed_point(_one_block(dict([fixed, seeded])), VOXEL, 4, ekw, incremental=True, before={})
    assert fp.as_set(rep["a_seed"]) == {(2, 1, 1)} and len(rep["b"]) == 0 and len(rep["a_other"]) == 0
    stale = ((2, 1, 1), (np.float32(0.3), 0, (-1, 0, 0)))
    after = _one_block(dict([fixed, stale]))
    rep = fp.fixed_point(after, VOXEL, 4, ekw, incremental=True, before=_copy(after))
    assert fp.as_set(rep["b_stale"]) == {(2, 1, 1)} and len(rep["b_other"]) == 0
    assert fp.as_set(rep["a_stale_source"]) == {(2, 1, 1)} and len(rep["a_other"]) == 0
    rep = fp.fixed_point(after, VOXEL, 4, ekw, incremental=True, before={})
    assert fp.as_set(rep["b_other"]) == {(2, 1, 1)} and fp.as_set(rep["a_other"]) == {(2, 1, 1)}


def test_incremental_mixed_class():
    """A target only the mixed-sign rule can still lower is class a_mixed, not a stale source or other."""
    ekw = dict(max_distance_m=2.0, default_distance_m=2.0, min_diff_m=0.0)
    blocks = _one_block({(1, 1, 1): (np.float32(0.05), 1, (0, 0, 0)), (2, 1, 1): (np.float32(-2.0), 0, (0, 0, 0))})
    rep = fp.fixed_point(blocks, VOXEL, 4, ekw, incremental=True, before={})
    assert fp.as_set(rep["a_mixed"]) == {(2, 1, 1)}
    assert len(rep["a_seed"]) == 0 and len(rep["a_stale_source"]) == 0 and len(rep["a_other"]) == 0


@pytest.mark.parametrize("case", ["parent_raised", "zero_parent", "parent_across"])
def test_stale_value_classes(case):
    """An unchanged value its parent no longer justifies: the parent's |d| rose on the same side (what only a
    raise does, and a raise resets the children: b_parent_raised), the voxel has no parent (b_zero_parent), or the
    parent crossed the surface (b_parent_across)."""
    ekw = dict(max_distance_m=2.0, default_distance_m=2.0, min_diff_m=0.0)
    p_then, p_now = {"parent_raised": (0.05, 0.15), "zero_parent": (0.05, 0.15), "parent_across": (0.05, -0.05)}[case]
    parent = (0, 0, 0) if case == "zero_parent" else (-1, 0, 0)
    v = ((2, 1, 1), (np.float32(np.float32(0.05) + np.float32(VOXEL)), 0, parent))
    before = _one_block(dict([((1, 1, 1), (np.float32(p_then), 1, (0, 0, 0))), v]))
    after = _one_block(dict([((1, 1, 1), (np.float32(p_now), 1, (0, 0, 0))), v]))
    rep = fp.fixed_point(after, VOXEL, 4, ekw, incremental=True, before=before)
    for c in ("b_parent_raised", "b_zero_parent", "b_parent_across", "b_stale", "b_other"):
        assert fp.as_set(rep[c]) == ({(2, 1, 1)} if c == "b_" + case else set()), (c, rep[c])


def test_checker_on_dijkstra_reference(wall):
    """The float64 shortest-path values themselves, rounded to float32, as an ESDF layer: they lie on the
    reference within its tolerance (no over / under), while the float32 rules, which hold the wavefront to its own
    arithmetic, see every voxel where the float64 path sum rounds differently from the float32 chain of steps:
    one ulp too high is lowerable (a), any difference is unjustified (b)."""
    blocks, _, _ = wall
    grid, dist, _ = fp.shortest_paths(blocks, VOXEL, VPS, EKW)
    dflt = np.float32(EKW["default_distance_m"])
    m = _copy(blocks)
    keys = [tuple(int(c) for c in k) for k in grid.block_keys]
    for i in np.nonzero(~grid.fixed)[0]:
        flat = grid.obs_flat[i]
        vox = m[keys[flat // grid.nv]]
        sign = np.float32(1.0) if grid.d[i] > 0 else np.float32(-1.0)
        vox["distance"][flat % grid.nv] = sign * (np.float32(dist[i]) if np.isfinite(dist[i]) else dflt)
    rep = fp.counts(fp.fixed_point(m, VOXEL, VPS, EKW, parents=False))
    dj = fp.counts(fp.dijkstra_check(m, VOXEL, VPS, EKW))
    print(rep, dj)
    assert dj["over"] == 0 and dj["under"] == 0
    assert rep["reached"] == 15423
    assert (rep["a"], rep["b"]) == (1163, 3128)
