"""Host-side checks of a quasi-Euclidean ESDF layer that do not depend on the order in which the
wavefront visited its voxels (plain numpy, float32, one IEEE operation at a time, like parity.py).

The device claims three things of every observed voxel once an update has converged, and each can be
read off the output alone:

 (a) no rule can still fire: for every source (observed, |d| < max_distance) and every target next to it
     (observed, not fixed), the same-sign tests and the mixed-sign test of k_esdf_lower are false;
 (b) every value is justified: an observed, non-fixed voxel that does not hold +-default_distance has a
     neighbour that reproduces it under the `same` or `mixed` rule of k_esdf_parents (with min_diff > 0:
     within min_diff; for incremental updates also under the unscaled seed rule of k_esdf_seed);
 (c) parents (batch, min_diff = 0): a reached voxel's parent is the first neighbour in table order that
     reproduces its value exactly.

A float64 shortest-path reference of the same operation (scipy's Dijkstra over each sign's voxels, from
a super-source joined to every fixed voxel with weight |d_fixed|) bounds the values from above, and
equals them on same-sign components that the mixed rule cannot lower.

Blocks are {block index (3 ints): ESDF voxels [vps^3]} as Layer.blocks() / OracleMap.blocks(1) return
them; voxels are named by their global voxel index."""
from __future__ import annotations

import math
from typing import Dict, Tuple

import numpy as np

F32 = np.float32

# src/utils/neighbor_tools.cc:24-30 (vbx_esdf.cu kOff): 6 faces, 12 edges, 8 corners, in this order
K_OFF = np.array([
    (-1, 0, 0), (1, 0, 0), (0, -1, 0), (0, 1, 0), (0, 0, -1), (0, 0, 1), (-1, -1, 0), (-1, 1, 0), (1, -1, 0),
    (1, 1, 0), (0, -1, -1), (0, -1, 1), (0, 1, -1), (0, 1, 1), (-1, 0, -1), (1, 0, -1), (-1, 0, 1), (1, 0, 1),
    (-1, -1, -1), (-1, -1, 1), (-1, 1, -1), (-1, 1, 1), (1, -1, -1), (1, -1, 1), (1, 1, -1), (1, 1, 1)], np.int32)

_BIAS = 1 << 20


def _cfg(cfg, name):
    return cfg[name] if isinstance(cfg, dict) else getattr(cfg, name)


def steps(voxel_size: float):
    """(scaled d1..d3 as vbx_esdf.cu computes them: float32(sqrt k) * float32(voxel_size), unscaled u1..u3)."""
    u = (F32(1.0), F32(math.sqrt(2.0)), F32(math.sqrt(3.0)))
    v = F32(voxel_size)
    return tuple(F32(x * v) for x in u), u


def step_of(k: int, table):
    return table[0] if k < 6 else (table[1] if k < 18 else table[2])


def signum(v: np.ndarray) -> np.ndarray:
    """signum() as a float32 (+0.0 for both zeros, like (float)signum_d(v))."""
    return np.where(v == 0, F32(0), np.where(v < 0, F32(-1), F32(1))).astype(F32)


def _pack(b: np.ndarray) -> np.ndarray:
    b = b.astype(np.int64) + _BIAS
    return (b[..., 0] << 42) | (b[..., 1] << 21) | b[..., 2]


class Grid:
    """The observed voxels of an ESDF layer and their neighbours across blocks."""

    def __init__(self, blocks: Dict[Tuple[int, int, int], np.ndarray], vps: int):
        self.vps = vps
        self.L = int(vps).bit_length() - 1
        assert 1 << self.L == vps
        keys = np.array(sorted(blocks), np.int32).reshape(-1, 3)
        self.block_keys = keys
        self.packed = _pack(keys)
        assert (np.diff(self.packed) > 0).all()
        nv = vps ** 3
        vox = np.concatenate([blocks[tuple(int(c) for c in k)] for k in keys]) if len(keys) else None
        self.nv = nv
        lin = np.arange(nv, dtype=np.int64)
        local = np.stack([lin & (vps - 1), (lin >> self.L) & (vps - 1), lin >> (2 * self.L)], 1)
        self.obs_flat = np.nonzero(vox["observed"] != 0)[0] if vox is not None else np.zeros(0, np.int64)
        o = self.obs_flat
        self.gidx = (keys[o // nv].astype(np.int64) * vps + local[o % nv]).astype(np.int64)
        self.d = vox["distance"][o].astype(F32) if vox is not None else np.zeros(0, F32)
        self.fixed = vox["fixed"][o] != 0 if vox is not None else np.zeros(0, bool)
        self.parent = vox["parent"][o].astype(np.int32) if vox is not None else np.zeros((0, 3), np.int32)
        # flat index -> position among the observed voxels (-1: unobserved)
        self._pos = np.full(len(keys) * nv, -1, np.int64)
        self._pos[o] = np.arange(o.size)

    @property
    def n(self) -> int:
        return self.d.size

    def neighbour(self, k: int) -> np.ndarray:
        """Position (among the observed voxels) of every observed voxel's neighbour at K_OFF[k]; -1 where that
        neighbour is unobserved or lies in a block that does not exist (a missing ESDF block holds no voxel)."""
        return self.lookup(self.gidx + K_OFF[k])

    def lookup(self, g: np.ndarray) -> np.ndarray:
        """Position (among the observed voxels) of the voxels with global indices g [n, 3]; -1 where none."""
        b = g >> self.L
        loc = g - (b << self.L)
        key = _pack(b)
        p = np.searchsorted(self.packed, key)
        p = np.minimum(p, max(len(self.packed) - 1, 0))
        hit = self.packed[p] == key if len(self.packed) else np.zeros(key.shape, bool)
        lin = loc[:, 0] | (loc[:, 1] << self.L) | (loc[:, 2] << (2 * self.L))
        out = np.full(g.shape[0], -1, np.int64)
        out[hit] = self._pos[p[hit] * self.nv + lin[hit]]
        return out


def _names(grid: Grid, mask: np.ndarray) -> np.ndarray:
    """Global indices of the voxels in `mask`, sorted."""
    g = grid.gidx[mask]
    return g[np.lexsort(g.T[::-1])] if g.size else g.reshape(0, 3)


def fixed_point(blocks, voxel_size: float, vps: int, cfg, incremental: bool = False, parents: bool = True,
                before=None) -> Dict:
    """Checks (a), (b) and (c) on a converged ESDF layer.  Returns the voxels that break each one (global
    indices, sorted):
      a          targets that a source could still lower
      b          observed, non-fixed voxels not at +-default_distance whose value no neighbour justifies
      c          reached voxels whose parent is not the first exact justifier in table order (None unless
                 parents and min_diff == 0; voxels with no exact justifier are left to (b))
    and, for incremental updates, the classes their exceptions fall in (`before`: the layer's blocks as they
    were before the update; a voxel is "unchanged" when it was observed then and holds the same value):
      a_seed          (a) at a voxel whose value the unscaled seed rule reproduces
      a_mixed         (a) otherwise, where only the mixed-sign rule fires
      a_stale_source  (a) otherwise, where every source that fires is unchanged: a source this update never
                      queued
      b_parent_raised (b) at an unchanged voxel whose stored parent's |d| rose in this update on the voxel's
                      side of the surface: a child the raise did not reset
      b_zero_parent   (b) otherwise, at an unchanged voxel with a zero parent (a seed value, cc:199, or a reset
                      one) that no raise can reach through parent pointers
      b_parent_across (b) otherwise, at an unchanged voxel whose stored parent lies on the other side of the
                      surface (a fixed voxel lowered through zero is not raised, cc:222-239, so its children
                      are not reset)
      b_stale         (b) otherwise, at an unchanged voxel: a value this update did not re-derive
      a_other, b_other  the rest"""
    grid = Grid(blocks, vps)
    (d1, d2, d3), (u1, u2, u3) = steps(voxel_size)
    md = F32(_cfg(cfg, "min_diff_m"))
    mx = F32(_cfg(cfg, "max_distance_m"))
    dflt = F32(_cfg(cfg, "default_distance_m"))
    d, fixed = grid.d, grid.fixed
    unchanged = np.zeros(grid.n, bool)
    parent_raised = np.zeros(grid.n, bool)
    jp, dp_now = np.full(grid.n, -1), np.zeros(grid.n, F32)
    if before is not None:
        prev = Grid(before, vps)

        def then(g):
            """Value before the update of the voxels at g (NaN where not observed then)."""
            j = prev.lookup(g)
            return np.where(j >= 0, prev.d[np.maximum(j, 0)] if prev.n else F32(0), F32(np.nan)).astype(F32)

        unchanged = then(grid.gidx).view(np.int32) == d.view(np.int32)
        # the stored parent's |d| rose on the voxel's side of the surface: only a raise does that, and a raise
        # resets every voxel whose parent points at the raised one (cc:349-356)
        gp = grid.gidx + grid.parent
        jp = grid.lookup(gp)
        dp_now = np.where(jp >= 0, d[np.maximum(jp, 0)], F32(np.nan))
        dp_then = then(gp)
        side = d > 0
        parent_raised = ((grid.parent != 0).any(1) & (jp >= 0) & ~np.isnan(dp_then)
                         & ((dp_now > 0) == side) & ((dp_then > 0) == side) & (np.abs(dp_now) > np.abs(dp_then)))
    target = ~fixed
    reached = target & (d != dflt) & (d != -dflt)
    fire = np.zeros(grid.n, bool)
    fire_same = np.zeros(grid.n, bool)
    fire_changed = np.zeros(grid.n, bool)
    justified = np.zeros(grid.n, bool)
    seeded = np.zeros(grid.n, bool)
    first = np.full(grid.n, -1, np.int64)
    sd = signum(d)
    ad = np.abs(d)
    for k in range(26):
        nb = grid.neighbour(k)
        has = nb >= 0
        s = np.where(has, nb, 0)
        ds = np.where(has, d[s], F32(0))
        src = has & (ds < mx) & (ds > -mx)     # a source, cc:387-390
        step = step_of(k, (d1, d2, d3))
        # (a) on the final values: the tests of k_esdf_lower
        out = (ds > 0) & (d > 0)
        ins = (ds <= 0) & (d <= 0)
        same_fire = (out & ((ds + step) + md < d)) | (ins & ((ds - step) - md > d))
        pot = ds - signum(ds) * step
        nv = np.where(signum(pot) == d, pot, sd * step).astype(F32)
        # the device applies the mixed-sign value only where it lowers |d| on the target's side (atomicMin)
        mixed_fire = (~out & ~ins & (np.abs(pot - d) > step) & ((nv > 0) == (d > 0))
                      & (nv.view(np.int32) < d.view(np.int32)))
        hit = src & target & (same_fire | mixed_fire)
        fire |= hit
        fire_same |= hit & same_fire
        fire_changed |= hit & ~unchanged[s]
        # (b) and (c): the `same` / `mixed` rules of k_esdf_parents (and the seed rule of k_esdf_seed)
        a = np.abs(ds) + step
        same_exact = (out | ins) & (a == ad)
        same_ok = same_exact if md == 0 else (out | ins) & (a <= ad) & (a + md >= ad)
        mixed_ok = ((d > 0) != (ds > 0)) & (sd * step == d)
        justified |= src & (same_ok | mixed_ok)
        first = np.where((first < 0) & src & (same_exact | mixed_ok), k, first)
        if incremental:
            u = step_of(k, (u1, u2, u3))
            seeded |= src & (signum(ds) == sd) & (np.abs(ds) < ad) & (ds + sd * u == d)
    unjust = reached & ~justified & ~seeded
    a_seed = fire & seeded
    a_mixed = fire & ~a_seed & ~fire_same
    a_stale = fire & ~a_seed & ~a_mixed & ~fire_changed & (before is not None)
    b_parent_raised = unjust & unchanged & parent_raised
    b_zero_parent = unjust & unchanged & ~b_parent_raised & (grid.parent == 0).all(1)
    b_parent_across = unjust & unchanged & ~b_parent_raised & ~b_zero_parent & (jp >= 0) & ((dp_now > 0) != (d > 0))
    b_stale = unjust & unchanged & ~b_parent_raised & ~b_zero_parent & ~b_parent_across
    rep = {"observed": grid.n, "reached": int(reached.sum()),
           "a": _names(grid, fire), "b": _names(grid, unjust), "c": None,
           "a_seed": _names(grid, a_seed), "a_mixed": _names(grid, a_mixed), "a_stale_source": _names(grid, a_stale),
           "a_other": _names(grid, fire & ~a_seed & ~a_mixed & ~a_stale),
           "b_parent_raised": _names(grid, b_parent_raised), "b_zero_parent": _names(grid, b_zero_parent),
           "b_parent_across": _names(grid, b_parent_across),
           "b_stale": _names(grid, b_stale), "b_other": _names(grid, unjust & ~unchanged)}
    if parents and md == 0:
        want = K_OFF[np.maximum(first, 0)]
        rep["c"] = _names(grid, reached & (first >= 0) & (grid.parent != want).any(1))
    return rep


CLASSES = ("a_seed", "a_mixed", "a_stale_source", "a_other", "b_parent_raised", "b_zero_parent", "b_parent_across",
           "b_stale", "b_other")


def counts(rep: Dict) -> Dict[str, int]:
    """Number of voxels in each list of a fixed_point() / dijkstra_check() report."""
    return {k: (len(v) if isinstance(v, np.ndarray) else v) for k, v in rep.items()}


def shortest_paths(blocks, voxel_size: float, vps: int, cfg):
    """Float64 least fixed point of the same-sign relaxation: per sign, Dijkstra over that sign's observed
    voxels (edges into non-fixed voxels only, weights the float32 steps widened to float64) from a
    super-source joined to every fixed voxel with weight |d_fixed|, limited to max_distance.  Returns
    (grid, distance per observed voxel: inf where unreached, component tainted by the mixed rule)."""
    from scipy.sparse import csr_matrix
    from scipy.sparse.csgraph import connected_components, dijkstra

    grid = Grid(blocks, vps)
    (d1, d2, d3), _ = steps(voxel_size)
    mx = F32(_cfg(cfg, "max_distance_m"))
    d, fixed = grid.d, grid.fixed
    inside = d <= 0
    n = grid.n
    rows, cols, wts = [], [], []
    mixable = np.zeros(n, bool)   # a non-fixed voxel next to a source of the other sign
    for k in range(26):
        nb = grid.neighbour(k)
        has = nb >= 0
        s = np.where(has, nb, 0)
        same = has & (inside[s] == inside)
        # edge s -> v (v's neighbour at offset k is s; the step is symmetric)
        e = same & ~fixed
        rows.append(s[e])
        cols.append(np.nonzero(e)[0])
        wts.append(np.full(int(e.sum()), float(step_of(k, (d1, d2, d3))), np.float64))
        mixable |= has & ~same & ~fixed & (d[s] < mx) & (d[s] > -mx)
    # node n: the super-source.  scipy keeps explicitly stored zeros of a sparse matrix as zero-weight edges,
    # so a fixed voxel at distance 0 is joined with weight 0 (not dropped).
    fx = np.nonzero(fixed)[0]
    und = csr_matrix((np.ones(sum(x.size for x in rows)), (np.concatenate(rows), np.concatenate(cols))), shape=(n, n))
    r, c, w = (np.concatenate(x) for x in (rows + [np.full(fx.size, n, np.int64)], cols + [fx],
                                            wts + [np.abs(d[fx].astype(np.float64))]))
    dist = np.full(n, np.inf)
    for sign_mask in (inside, ~inside):
        keep = np.append(sign_mask, True)
        ok = keep[r] & keep[c]
        g = csr_matrix((w[ok], (r[ok], c[ok])), shape=(n + 1, n + 1))
        sp = dijkstra(g, directed=True, indices=n, limit=float(mx))
        dist[sign_mask] = sp[:n][sign_mask]
    # same-sign components (undirected) that hold a voxel the mixed rule can lower
    _, comp = connected_components(und, directed=False)
    tainted = np.isin(comp, np.unique(comp[mixable]))
    return grid, dist, tainted


def tolerance(dist: np.ndarray, voxel_size: float, cfg) -> np.ndarray:
    """Accumulated float32 rounding along a path of `hops` steps: 2 * hops * ulp(max_distance) (+ min_diff
    per hop, which a relaxation may leave unclaimed).  A path to distance D has at most D / d1 + 1 hops
    (every step is at least d1; one more for the fixed voxel's own value)."""
    (d1, _, _), _ = steps(voxel_size)
    mx = F32(_cfg(cfg, "max_distance_m"))
    md = float(_cfg(cfg, "min_diff_m"))
    hops = np.floor(np.where(np.isfinite(dist), dist, float(mx)) / float(d1)) + 2
    return hops * (2 * float(np.spacing(mx)) + md)


def dijkstra_check(blocks, voxel_size: float, vps: int, cfg) -> Dict:
    """Batch updates: |d| <= least fixed point + tolerance on every non-fixed observed voxel the reference
    reaches ("over"), and |d| >= least fixed point - tolerance (>= max_distance - tolerance where it reaches
    none) on the components the mixed rule cannot lower ("under")."""
    grid, dist, tainted = shortest_paths(blocks, voxel_size, vps, cfg)
    tol = tolerance(dist, voxel_size, cfg)
    ad = np.abs(grid.d.astype(np.float64))
    mx = float(F32(_cfg(cfg, "max_distance_m")))
    nonfixed = ~grid.fixed
    fin = np.isfinite(dist)
    over = nonfixed & fin & (ad > dist + tol)
    under = nonfixed & ~tainted & np.where(fin, ad < dist - tol, ad < mx - tol)
    return {"compared": int((nonfixed & fin).sum()), "clean": int((nonfixed & ~tainted).sum()),
            "over": _names(grid, over), "under": _names(grid, under)}


def as_set(names: np.ndarray):
    return {tuple(int(v) for v in g) for g in names}
