"""Host-side checks of a full-Euclidean ESDF layer (EsdfIntegrator::Config::full_euclidean_distance) that do not
depend on the order in which the wavefront visited its voxels (plain numpy, float32, one IEEE operation at a time,
restating the full-Euclidean branch of k_esdf_lower).

In full-Euclidean mode a source s with parent p_s offers its neighbour t = s + dir the parent p_s - dir and the step
    fmul(voxel_size, fsub(sqrtf(|p_s - dir|^2), sqrtf(|p_s|^2)))
(esdf_integrator.cc:414-426; the components are integers, so each squared norm is exact and each norm one correctly
rounded sqrtf); a candidate with a negative step is skipped.  The device keeps (distance, parent) in one 64-bit word
and lowers it with a signed 64-bit atomicMin: the distance's int32 bit pattern in the high 32 bits, the parent code
(component + 512, 10 bits each, x low) in the low 32.  The checks below compare words in THAT order, not in float
order: for two inside values it is the one nearer zero that is smaller, -0.0 (int32 0x80000000) is the smallest
word any value can have, +0.0 lies above every negative value, and equal distances compare by parent code.

Checks, reading the output layer (and for incremental updates the layer before the update):
 (a) nothing can fire: for every source (observed, |d| < max_distance) and every observed, non-fixed neighbour, no
     candidate of the same-sign or the mixed-sign rule meets the rule's condition and is a strictly smaller word
     than the target's;
 (r) roots: every rule sets new_parent = p_s - dir, so root = v + parent is the same voxel along a whole chain, and
     chains start only at fixed voxels (batch, default_distance >= max_distance) or at seeded voxels (parent 0,
     incremental).  Every reached voxel (observed, not fixed, not at +-default) is classified by its root;
 (t) telescoping: along a same-sign chain the exact steps sum to voxel_size * |parent|, so
         |d(v) - (d(root) + sign(v) * voxel_size * |parent(v)|)| <= tolerance(parent)   (see tolerance())
     for every voxel whose root is a fixed voxel of its own sign;
 (e) a float64 Euclidean reference: min over the fixed voxels f of v's sign of |d(f)| + voxel_size * |v - f|,
     brute force.  The 26-neighbour vector propagation is not an exact EDT at Voronoi boundaries, so |d| - EDT is
     reported as a distribution; |d| >= EDT - tolerance follows from (t).
Voxels are named by their global voxel index, like tests/esdf_fixed_point.py."""
from __future__ import annotations

from typing import Dict

import numpy as np

from tests.esdf_fixed_point import F32, K_OFF, Grid, _cfg, _names, signum, steps

BIAS = 512
U = 2.0 ** -24          # unit roundoff of float32


def parent_code(parent: np.ndarray) -> np.ndarray:
    """fe_pack's low 32 bits (no masking, like the device: a component outside [-512, 511] spills over)."""
    p = parent.astype(np.int64) + BIAS
    return (p[..., 0] | (p[..., 1] << 10) | (p[..., 2] << 20)) & 0xFFFFFFFF


def parent_decode(code: np.ndarray) -> np.ndarray:
    """fe_parent: the parent that a code unpacks to."""
    c = np.asarray(code, np.int64)
    return np.stack([(c & 1023) - BIAS, ((c >> 10) & 1023) - BIAS, ((c >> 20) & 1023) - BIAS], -1).astype(np.int32)


def parent_ok(parent: np.ndarray) -> np.ndarray:
    """fe_parent_ok: every component in [-512, 511]."""
    return ((parent >= -BIAS) & (parent < BIAS)).all(-1)


def word(d: np.ndarray, parent: np.ndarray) -> np.ndarray:
    """The device's 64-bit (distance, parent) word as a signed int64: words compare in THIS order (not float order)."""
    hi = np.asarray(d, F32).view(np.int32).astype(np.int64)
    return (hi << 32) | parent_code(parent)


def _sqrt_norm(p: np.ndarray) -> np.ndarray:
    """norm3 of an integer vector: the squared norm is exact in float32 for |components| < 2048, one sqrtf."""
    n2 = (p.astype(np.int64) ** 2).sum(-1)
    return np.sqrt(n2.astype(F32)).astype(F32)


def fe_step(voxel_size: float, p_src: np.ndarray, k: int):
    """(new parent, step) of a source with parent p_src towards K_OFF[k], as k_esdf_lower computes them."""
    newp = (p_src - K_OFF[k]).astype(np.int32)
    step = (F32(voxel_size) * (_sqrt_norm(newp) - _sqrt_norm(p_src)).astype(F32)).astype(F32)
    return newp, step


def rounded_direction(parent: np.ndarray) -> np.ndarray:
    """roundf(unit3(parent)) per component (the raise test of cc:339-347 / k_esdf_raise); zero for parent 0."""
    p = parent.astype(F32)
    z = (p[:, 0] * p[:, 0] + (p[:, 1] * p[:, 1] + p[:, 2] * p[:, 2])).astype(F32)
    s = np.sqrt(z).astype(F32)
    u = np.where(z[:, None] > 0, p / np.where(s > 0, s, F32(1))[:, None], p).astype(F32).astype(np.float64)
    return (np.sign(u) * np.floor(np.abs(u) + 0.5)).astype(np.int32)   # roundf: half away from zero


def tolerance(parent_len2: np.ndarray, voxel_size: float, cfg) -> np.ndarray:
    """Bound on |d(v) - (d(root) + sign * voxel_size * |parent|)| for a chain of float32 steps from the root.

    Let the chain be p_0 = 0 (the root), p_1, ..., p_n = parent(v), each link one 26-neighbourhood offset, and
    s_i = sqrtf(|p_i|^2).  Hop i adds fmul(vs, fsub(s_i, s_{i-1})) with one fadd (fsub inside).
      * The s_i telescope: the exact sum of s_i - s_{i-1} is s_n, which is |p_n| within U * |p_n|.
      * fsub and fmul each round relative to their result, so all steps together add at most
        2U * vs * sum(s_i - s_{i-1}) = 2U * vs * s_n.
      * A hop with a zero step adds exactly 0, so only hops with a positive step round in the fadd.  A step is
        positive only if the integer |p_i|^2 rises, and it starts at 0: at most |p_n|^2 such hops.  Every chain
        voxel but the last was a source (|d| < max_distance) and the last was lowered from at most
        default_distance, so every fadd result lies within M = max(max_distance, default_distance) and rounds
        by at most ulp(M) / 2.
    tolerance = |p|^2 * ulp(M) / 2 + 3U * vs * |p| (+ a 1 % margin on the whole for the second-order terms)."""
    vs = float(F32(voxel_size))
    m = max(float(F32(_cfg(cfg, "max_distance_m"))), float(F32(_cfg(cfg, "default_distance_m"))))
    n2 = parent_len2.astype(np.float64)
    return 1.01 * (n2 * float(np.spacing(F32(m))) / 2 + 3 * U * vs * np.sqrt(n2))


ROOT_CLASSES = ("r_fixed_same", "r_fixed_other", "r_seeded", "r_unit", "r_other")
A_CLASSES = ("a_seed", "a_mixed", "a_stale_source", "a_other")
STALE_CLASSES = ("s_parent_raised", "s_crossed", "s_rest")


def fe_check(blocks, voxel_size: float, vps: int, cfg, incremental: bool = False, before=None) -> Dict:
    """(a), (r) and (t) on a converged full-Euclidean ESDF layer.  Returns the voxels in each list (global
    indices, sorted):
      a               targets some candidate could still lower (fire, below); split into
        a_seed          (incremental) the target's value is the unscaled seed step from a neighbour (k_esdf_seed)
        a_mixed         otherwise, only the mixed-sign rule fires
        a_stale_source  (incremental) otherwise, every source that fires is unchanged: one the update never queued
        a_other         the rest
      range           voxels whose parent does not round-trip through the 10-bit code (k_esdf_fe_pack fails on them)
      r_fixed_same    reached voxels whose root is a fixed voxel of their sign
      r_fixed_other   ... a fixed voxel of the other sign (the chain crossed the surface through the mixed rule)
      r_seeded        ... a non-fixed voxel with parent 0 (a seeded voxel, or the voxel itself; incremental)
      r_unit          ... otherwise the voxel's parent is a unit offset (a quasi-Euclidean parent)
      r_other         the rest
      t               r_fixed_same voxels off the telescoping identity by more than tolerance()
    and, for incremental updates, the reached voxels an update left unchanged (same value and parent) whose root is
    no longer a fixed voxel of their sign:
      s_parent_raised   the neighbour their rounded parent direction points at (the raise test of cc:339-347) is
                        further from the surface on the voxel's side than before the update: a child the raise
                        should have reset
      s_crossed         otherwise, the root is a fixed voxel of the other sign or lies on the other side
      s_rest            the rest
    Counts: observed, reached, and t_max_err (largest telescoping error over r_fixed_same)."""
    grid = Grid(blocks, vps)
    _, (u1, u2, u3) = steps(voxel_size)
    md = F32(_cfg(cfg, "min_diff_m"))
    mx = F32(_cfg(cfg, "max_distance_m"))
    dflt = F32(_cfg(cfg, "default_distance_m"))
    d, fixed, par = grid.d, grid.fixed, grid.parent
    n = grid.n
    w_t = word(d, par)
    unchanged = np.zeros(n, bool)
    prev = None
    if before is not None:
        prev = Grid(before, vps)
        j = prev.lookup(grid.gidx)
        jj = np.maximum(j, 0)
        if prev.n:
            unchanged = (j >= 0) & (prev.d[jj].view(np.int32) == d.view(np.int32)) & (prev.parent[jj] == par).all(1)
    target = ~fixed
    reached = target & (d != dflt) & (d != -dflt)
    fire = np.zeros(n, bool)
    fire_same = np.zeros(n, bool)
    fire_changed = np.zeros(n, bool)
    seeded_val = np.zeros(n, bool)
    sd = signum(d)
    for k in range(26):
        nb = grid.neighbour(k)             # the voxel at v + K_OFF[k] is the source s; v = s - K_OFF[k]
        has = nb >= 0
        s = np.where(has, nb, 0)
        ds = np.where(has, d[s], F32(0))
        src = has & (ds < mx) & (ds > -mx)
        # s reaches v in direction -K_OFF[k]: index of that offset in the table
        kk = int(np.nonzero((K_OFF == -K_OFF[k]).all(1))[0][0])
        newp, step = fe_step(voxel_size, par[s], kk)
        ok = src & target & (step >= 0) & parent_ok(newp)
        out = (ds > 0) & (d > 0)
        ins = (ds <= 0) & (d <= 0)
        same_c = (out & (((ds + step) + md) < d)) | (ins & (((ds - step) - md) > d))
        same_v = np.where(out, ds + step, ds - step).astype(F32)
        pot = (ds - (signum(ds) * step).astype(F32)).astype(F32)
        nv = np.where(signum(pot) == d, pot, (sd * step).astype(F32)).astype(F32)
        mixed_c = ~out & ~ins & (np.abs((pot - d).astype(F32)) > step) & ((nv > 0) == (d > 0))
        cand = np.where(same_c, same_v, nv).astype(F32)
        hit = ok & (same_c | mixed_c) & (word(cand, newp) < w_t)
        fire |= hit
        fire_same |= hit & same_c
        fire_changed |= hit & ~unchanged[s]
        if incremental:
            u = u1 if kk < 6 else (u2 if kk < 18 else u3)
            seeded_val |= src & (signum(ds) == sd) & (np.abs(ds) < np.abs(d)) & ((ds + sd * u).astype(F32) == d)
    a_seed = fire & seeded_val
    a_mixed = fire & ~a_seed & ~fire_same
    a_stale = fire & ~a_seed & ~a_mixed & ~fire_changed & (before is not None)
    a_other = fire & ~a_seed & ~a_mixed & ~a_stale
    # (r) roots
    jr = grid.lookup(grid.gidx + par)
    jr0 = np.maximum(jr, 0)
    found = jr >= 0
    root_fixed = found & fixed[jr0]
    same_side = (d[jr0] > 0) == (d > 0)
    r_fixed_same = reached & root_fixed & same_side
    r_fixed_other = reached & root_fixed & ~same_side
    r_seeded = reached & ~root_fixed & found & (par[jr0] == 0).all(1)
    unit = (np.abs(par) <= 1).all(1) & (par != 0).any(1)
    r_unit = reached & ~root_fixed & ~r_seeded & unit
    r_other = reached & ~root_fixed & ~r_seeded & ~r_unit
    # (t) telescoping, float64
    n2 = (par.astype(np.int64) ** 2).sum(1)
    pred = d[jr0].astype(np.float64) + np.where(d > 0, 1.0, -1.0) * float(F32(voxel_size)) * np.sqrt(n2)
    err = np.abs(d.astype(np.float64) - pred)
    t_bad = r_fixed_same & (err > tolerance(n2, voxel_size, cfg))
    rep = {"observed": n, "reached": int(reached.sum()),
           "t_max_err": float(err[r_fixed_same].max()) if r_fixed_same.any() else 0.0,
           "a": _names(grid, fire), "a_seed": _names(grid, a_seed), "a_mixed": _names(grid, a_mixed),
           "a_stale_source": _names(grid, a_stale), "a_other": _names(grid, a_other),
           "range": _names(grid, ~parent_ok(par)),
           "r_fixed_same": _names(grid, r_fixed_same), "r_fixed_other": _names(grid, r_fixed_other),
           "r_seeded": _names(grid, r_seeded), "r_unit": _names(grid, r_unit), "r_other": _names(grid, r_other),
           "t": _names(grid, t_bad)}
    if prev is not None:
        gone = reached & unchanged & ~r_fixed_same
        # the neighbour the raise test takes for the voxel's parent
        pn = grid.gidx + rounded_direction(par)
        jn = grid.lookup(pn)
        jp = prev.lookup(pn)
        dn_now = np.where(jn >= 0, d[np.maximum(jn, 0)], F32(np.nan))
        dn_then = np.where(jp >= 0, prev.d[np.maximum(jp, 0)] if prev.n else F32(0), F32(np.nan))
        side = d > 0
        raised = ((par != 0).any(1) & (jn >= 0) & (jp >= 0) & ((dn_now > 0) == side) & ((dn_then > 0) == side)
                  & (np.abs(dn_now) > np.abs(dn_then)))
        s_raised = gone & raised
        crossed = gone & ~s_raised & found & ~same_side
        rep.update({"s_parent_raised": _names(grid, s_raised), "s_crossed": _names(grid, crossed),
                    "s_rest": _names(grid, gone & ~s_raised & ~crossed)})
    return rep


def counts(rep: Dict) -> Dict:
    return {k: (len(v) if isinstance(v, np.ndarray) else v) for k, v in rep.items()}


def euclidean(blocks, voxel_size: float, vps: int, cfg, max_pairs: float = 5e8):
    """(e): the float64 weighted Euclidean distance of every observed voxel whose root is a fixed voxel of its sign,
    min over the fixed voxels f of that sign of |d(f)| + voxel_size * |v - f|, by chunked brute force.  Returns None
    where voxels x fixed voxels exceeds `max_pairs` (not affordable); else a dict with the distribution of
    |d| - EDT (metres) and the voxels below EDT by more than tolerance() ("under")."""
    grid = Grid(blocks, vps)
    d, fixed, par = grid.d, grid.fixed, grid.parent
    jr = grid.lookup(grid.gidx + par)
    jr0 = np.maximum(jr, 0)
    dflt = F32(_cfg(cfg, "default_distance_m"))
    reached = ~fixed & (d != dflt) & (d != -dflt)
    rooted = reached & (jr >= 0) & fixed[jr0] & ((d[jr0] > 0) == (d > 0))
    vs = float(F32(voxel_size))
    edt = np.full(grid.n, np.inf)
    pairs = 0
    for side in (d > 0, d <= 0):
        v = np.nonzero(rooted & side)[0]
        f = np.nonzero(fixed & side)[0]
        pairs += v.size * f.size
    if pairs > max_pairs:
        return None
    for side in (d > 0, d <= 0):
        v = np.nonzero(rooted & side)[0]
        f = np.nonzero(fixed & side)[0]
        if v.size == 0 or f.size == 0:
            continue
        fg = grid.gidx[f].astype(np.float64)
        fd = np.abs(d[f].astype(np.float64))
        chunk = max(1, int(4e6 // f.size))
        for i in range(0, v.size, chunk):
            vi = v[i:i + chunk]
            diff = grid.gidx[vi].astype(np.float64)[:, None, :] - fg[None]
            edt[vi] = (fd[None] + vs * np.sqrt((diff ** 2).sum(-1))).min(1)
    ad = np.abs(d.astype(np.float64))
    n2 = (par.astype(np.int64) ** 2).sum(1)
    tol = tolerance(n2, voxel_size, cfg)
    ex = (ad - edt)[rooted]
    q = np.quantile(ex, [0.5, 0.99, 0.999]) if ex.size else np.zeros(3)
    return {"compared": int(rooted.sum()), "under": _names(grid, rooted & (ad < edt - tol)),
            "exact": int((np.abs(ad - edt)[rooted] <= tol[rooted]).sum()),
            "over_tol": int((ad - edt > tol)[rooted].sum()), "over_voxel": int((ad - edt > vs)[rooted].sum()),
            "median": float(q[0]), "p99": float(q[1]), "p999": float(q[2]),
            "max": float(ex.max()) if ex.size else 0.0, "edt": edt, "grid": grid}


def as_set(names: np.ndarray):
    return {tuple(int(v) for v in g) for g in names}


# ------------------------------------------------------------------ synthetic TSDF scenes
# Every listed voxel has weight 1 and a TSDF distance chosen so that the fixed set (|tsdf| < min_distance) is exactly
# the voxels intended; every other voxel of their blocks has weight 0 (unobserved for the ESDF).
SYN_VOXEL, SYN_FREE, SYN_MIN_DISTANCE = 0.1, 0.2, 0.05
SYN_EKW = dict(max_distance_m=2.0, default_distance_m=2.0, min_distance_m=SYN_MIN_DISTANCE, min_diff_m=0.0,
               multi_queue=1, full_euclidean_distance=1)
HAIRPIN_L = 6


def _cube(r=8):
    a = np.arange(-r, r)
    return np.stack(np.meshgrid(a, a, a, indexing="ij"), -1).reshape(-1, 3).astype(np.int64)


def synthetic(name: str):
    """(global voxel indices [m, 3], TSDF distances [m]) of a synthetic scene."""
    if name in ("point", "point_inside", "two_points"):
        g = _cube()
        inside = name == "point_inside"
        d = np.full(len(g), -SYN_FREE if inside else SYN_FREE, F32)
        fixed = {"point": {(-3, 2, 1): 0.013}, "point_inside": {(-3, 2, 1): -0.0},
                 "two_points": {(-4, -1, 0): 0.005, (3, 2, -2): 0.04}}[name]
        for v, fd in fixed.items():
            d[((g == v).all(1))] = F32(fd)
        return g, d
    if name == "plane":      # z = 0 fixed outside, z = -1 fixed inside, free voxels above / below
        g = _cube()
        z = g[:, 2]
        d = np.where(z >= 1, SYN_FREE, np.where(z <= -2, -SYN_FREE, np.where(z == 0, 0.02, -0.03))).astype(F32)
        return g, d
    if name == "tilted":     # fixed within one voxel of the plane x + 2y + 3z = 0: no two free voxels of opposite
        g = _cube()          # sign are neighbours (a corner step changes t by 6 / sqrt(14) < 2)
        t = (g @ np.array([1.0, 2.0, 3.0])) / np.sqrt(14.0)
        d = np.where(np.abs(t) < 1.0, 0.04 * t, np.where(t > 0, SYN_FREE, -SYN_FREE)).astype(F32)
        return g, d
    if name == "hairpin":    # a one-voxel path out along +x, over 3 in y, and back along -x (see the GPU test)
        L = HAIRPIN_L
        g = ([(x, 0, 0) for x in range(L + 1)] + [(L, y, 0) for y in (1, 2, 3)] + [(x, 3, 0) for x in range(L - 1, -1, -1)])
        g = np.array(g, np.int64)
        d = np.full(len(g), SYN_FREE, F32)
        d[0] = F32(0.01)
        return g, d
    raise KeyError(name)


def tsdf_blocks(g: np.ndarray, d: np.ndarray, vps: int):
    """(block indices [n, 3] int32, TSDF voxels [n, vps^3]) holding distance d and weight 1 at voxels g."""
    from oracle import pyoracle as po
    b = np.floor_divide(g, vps)
    keys, inv = np.unique(b, axis=0, return_inverse=True)
    inv = inv.reshape(-1)
    loc = g - b * vps
    lin = loc[:, 0] + vps * (loc[:, 1] + vps * loc[:, 2])
    vox = np.zeros((len(keys), vps ** 3), po.TSDF_DTYPE)
    vox["distance"][inv, lin] = d
    vox["weight"][inv, lin] = 1.0
    return keys.astype(np.int32), vox


def oracle_layer(lib, g, d, vps, ekw, voxel=SYN_VOXEL):
    """The oracle map of a synthetic TSDF layer after a batch ESDF update."""
    from oracle import pyoracle as po
    idx, vox = tsdf_blocks(g, d, vps)
    omap = po.OracleMap(lib, po.TsdfConfig(default_truncation_distance=SYN_FREE, integrator_threads=1), voxel, vps)
    omap.esdf_create(po.EsdfConfig(**ekw))
    for i, v in zip(idx, vox):
        omap.deserialize_block(i, v.view(np.uint32), 0)
    omap.esdf_update(batch=True)
    return omap
