"""-m gpu: the TSDF apply (record sort, k_apply_prep, k_apply) driven through vbx_debug_apply with chosen
update sequences and prior voxel states, against a sequential NumPy restatement of updateTsdfVoxel
(tsdf_integrator.cc:186-208).

k_apply picks one of about ten arithmetic paths per run, 128-record step or 32-record chunk, and each one
claims the sequential result bit for bit.  Every case here targets some of them: it compares all 12 bytes
of every voxel of the touched blocks with the reference, and asserts that the apply-path counters show
the paths the case was built for.  test_every_path_ran checks that the cases together reach every path."""
import ctypes as C

import numpy as np
import pytest

import voxblox_b200 as vb

pytestmark = pytest.mark.gpu

F = np.float32
EPS = F(1e-6)       # kFloatEpsilon, core/common.h:139-140
VPS = 16
NV = VPS ** 3
TILE = 256          # records per short-run tile of k_apply
SHORT = 32          # kShortRun: longer runs go to one warp each
PATHS = vb.api.TsdfIntegratorBase.APPLY_PATHS


# ------------------------------------------------------------------------------------------- reference
def _blend(c1, w1, c2, w2):
    """Color::blendTwoColors (core/common.h:105-125) in float32; round() is half away from zero, here on
    non-negative values: floor(x + 0.5) in double."""
    tot = w1 + w2
    a = (w1 / tot)[:, None]
    b = (w2 / tot)[:, None]
    v = c1.astype(F) * a + c2.astype(F) * b
    return (np.floor(v.astype(np.float64) + 0.5).astype(np.int64) & 0xFF).astype(np.uint8)


def reference_apply(vox, rec_vox, sdf, w, rgba, T, max_weight):
    """updateTsdfVoxel applied in record order: vox (TSDF_DTYPE, flat) is updated in place; record r goes to
    vox[rec_vox[r]].  Vectorised across voxels, sequential along each voxel's chain."""
    T, MW = F(T), F(max_weight)
    order = np.argsort(rec_vox, kind="stable")
    rv = rec_vox[order]
    first = np.r_[0, np.flatnonzero(rv[1:] != rv[:-1]) + 1]
    lens = np.diff(np.r_[first, len(rv)])
    rank = np.arange(len(rv)) - np.repeat(first, lens)
    by_rank = np.argsort(rank, kind="stable")
    starts = np.r_[0, np.cumsum(np.bincount(rank, minlength=int(lens.max()) if len(lens) else 0))]
    D, W, Col = vox["distance"], vox["weight"], vox["color"]
    with np.errstate(all="ignore"):
        for k in range(len(starts) - 1):
            r = order[by_rank[starts[k]:starts[k + 1]]]
            v = rec_vox[r]
            d, wt, s, u = D[v], W[v], sdf[r], w[r]
            nw = wt + u
            ok = ~(nw < EPS)
            ns = (s * u + d * wt) / nw
            bl = ok & (np.abs(s) < T)
            if bl.any():
                Col[v[bl]] = _blend(Col[v[bl]], wt[bl], rgba[r[bl]], u[bl])
            # std::min(T, x) / std::max(-T, x) return their first argument on NaN
            nd = np.where(ns > 0, np.where(ns < T, ns, T), np.where(-T < ns, ns, -T)).astype(F)
            D[v[ok]] = nd[ok]
            W[v[ok]] = np.where(nw < MW, nw, MW)[ok]


# ---------------------------------------------------------------------------------------------- cases
class Case:
    """Blocks (n_blocks along x) with prior voxels, and records in application order."""

    def __init__(self, T, max_weight, n_blocks=1):
        self.T, self.max_weight = F(T), F(max_weight)
        self.prior = np.zeros(n_blocks * NV, vb.api.TSDF_DTYPE)
        self.vox, self.sdf, self.w, self.rgba = [], [], [], []

    def run(self, v, sdf, w, rgba=None):
        """A chain of updates of flat voxel v (block v // NV)."""
        sdf = np.asarray(sdf, F).reshape(-1)
        n = len(sdf)
        w = np.broadcast_to(np.asarray(w, F), (n,))
        if rgba is None:
            rgba = np.stack([(np.arange(n) * 37 + v) % 256, (np.arange(n) * 11) % 256,
                             np.full(n, 200), np.full(n, 255)], 1)
        self.vox.append(np.full(n, v, np.int64))
        self.sdf.append(sdf)
        self.w.append(np.array(w, F))
        self.rgba.append(np.asarray(rgba, np.uint8).reshape(n, 4))
        return self

    def arrays(self):
        cat = lambda xs, dt: np.concatenate(xs).astype(dt) if xs else np.zeros(0, dt)
        return (cat(self.vox, np.int64), cat(self.sdf, F), cat(self.w, F),
                np.concatenate(self.rgba) if self.rgba else np.zeros((0, 4), np.uint8))


def _layer(T, max_weight, n_blocks, vps=VPS, max_updates=0):
    cfg = vb.TsdfIntegratorConfig(default_truncation_distance=float(T), max_weight=float(max_weight),
                                  integrator_threads=1)
    layer = vb.Layer(0.1, vps, engine_options=vb.EngineOptions(max_updates_per_pass=max_updates))
    integ = vb.TsdfIntegratorFactory.create("simple", cfg, layer)
    idx = np.zeros((n_blocks, 3), np.int32)
    idx[:, 0] = np.arange(n_blocks)
    return layer, integ, idx


def debug_apply(layer, idx, rec_block, rec_voxel, sdf, w, rgba):
    ctx = layer._ctx
    paths = np.zeros(16, np.uint64)
    idx = np.ascontiguousarray(idx, np.int32)
    rb = np.ascontiguousarray(rec_block, np.uint32)
    rv = np.ascontiguousarray(rec_voxel, np.uint32)
    sdf, w = np.ascontiguousarray(sdf, F), np.ascontiguousarray(w, F)
    rgba = np.ascontiguousarray(rgba, np.uint8)
    ctx.check(ctx.lib.vbx_debug_apply(ctx.handle, idx.ctypes.data, C.c_uint32(len(idx)), len(sdf), rb.ctypes.data,
                                      rv.ctypes.data, sdf.ctypes.data, w.ctypes.data, rgba.ctypes.data,
                                      paths.ctypes.data), "vbx_debug_apply")
    return {k: int(v) for k, v in zip(PATHS, paths)}


def check_case(case, max_updates=0):
    """Device vs reference over every voxel of the case's blocks (all 12 bytes); returns the path counts
    and the reference's voxels."""
    nb = len(case.prior) // NV
    layer, integ, idx = _layer(case.T, case.max_weight, nb, max_updates=max_updates)
    layer.insertBlocks(idx, case.prior.reshape(nb, NV))
    vox, sdf, w, rgba = case.arrays()
    paths = debug_apply(layer, idx, vox // NV, vox % NV, sdf, w, rgba)
    ref = case.prior.copy()
    reference_apply(ref, vox, sdf, w, rgba, case.T, case.max_weight)
    got, _ = layer.getBlocks(idx)
    got = np.ascontiguousarray(got).reshape(-1)
    bad = np.flatnonzero((got.view(np.uint8).reshape(-1, 12) != ref.view(np.uint8).reshape(-1, 12)).any(axis=1))
    assert len(bad) == 0, (f"{len(bad)} voxels differ; first {bad[:5]}: device {got[bad[:5]]} reference {ref[bad[:5]]}"
                           f" prior {case.prior[bad[:5]]}")
    return paths, ref


RAN = {}   # case name -> path counts of its run (test_every_path_ran)


def _expect(name, paths, want, zero=()):
    RAN[name] = paths
    print(name, paths)
    for k in want:
        assert paths[k] > 0, (name, k, paths)
    for k in zero:
        assert paths[k] == 0, (name, k, paths)


# -- run lengths and positions
def case_run_lengths():
    c = Case(0.3, 10000.0, n_blocks=2)
    rng = np.random.default_rng(1)
    v = 0
    for n in (1, 31, 32, 33, 127, 128, 129, 255, 256, 257, 1023, 1024, 1025, 4097, 40000):
        c.prior[v] = (F(rng.uniform(-0.3, 0.3)), F(rng.uniform(0, 20)), (10, 20, 30, 255))
        c.run(v, rng.uniform(-0.6, 0.9, n), rng.uniform(0.0, 2.0, n))
        v += 1
    return c, ["long_runs", "short_runs", "chunk_exact"]


def case_tile_offsets():
    """Runs that start at tile offsets 0, 1, 224 and 255 of the short-run phase, and short runs that cross a
    tile's end by exactly one record: the layout of the sorted records is set by the voxels' order."""
    c = Case(0.3, 10000.0)
    rng = np.random.default_rng(2)
    lens = []
    # tile 0, all short runs: one at offset 0 (len 1), one at 1 (len 31), six of 32 filling [32, 224), one at 224
    # (len 31), one at 255 crossing by 1
    lens += [1, 31] + [32] * 6 + [31, 2]
    # tile 1 (from 257): a long run fills to offset 255, then a run of 32 that crosses by 31 records
    lens += [255 - 1, 32]
    # tile 2 (from 512 + 31): short runs; the last one crosses by exactly one record
    pos = 512 + 31
    while pos + 20 < 768 - 19:
        lens.append(20)
        pos += 20
    lens.append(768 + 1 - pos)
    # a long run that starts in the middle of a tile, then short runs after it
    lens += [100, 5, 7]
    starts = np.cumsum([0] + lens[:-1])
    assert [int(starts[k]) % TILE for k in (0, 1, 8, 9)] == [0, 1, 224, 255] and lens[9] == 2
    for v, n in enumerate(lens):
        c.prior[v] = (F(0.1), F(2.0), (1, 2, 3, 4))
        c.run(v, rng.uniform(-0.4, 0.5, n), rng.uniform(0.1, 1.0, n))
    return c, ["short_runs", "short_crossed", "long_runs"]


def case_runs_of_33_fill_the_pass():
    """Enough runs of 33 records (one over kShortRun) to fill max_updates_per_pass: each warp takes many long-run
    tickets."""
    max_updates = 1 << 20
    n_runs = max_updates // 33
    nb = (n_runs + NV - 1) // NV
    c = Case(0.25, 10000.0, n_blocks=nb)
    rng = np.random.default_rng(3)
    c.prior["distance"][:n_runs] = F(0.25)
    c.prior["weight"][:n_runs] = rng.integers(0, 50, n_runs).astype(F)
    sdf = rng.choice(np.array([0.5, 0.25, 0.1, -0.3], F), size=(n_runs, 33), p=[0.7, 0.1, 0.1, 0.1])
    w = rng.integers(1, 4, (n_runs, 33)).astype(F)
    c.vox = [np.repeat(np.arange(n_runs), 33)]
    c.sdf, c.w = [sdf.reshape(-1)], [w.reshape(-1)]
    c.rgba = [rng.integers(0, 256, (n_runs * 33, 4)).astype(np.uint8)]
    return c, ["long_runs"], max_updates


# -- free space on a voxel at +T: the step and chunk weight chains
def case_step_paths():
    """Free-space runs (sdf >= T) on voxels at +T, decided a whole 128-record step at a time."""
    c = Case(0.25, 10000.0)
    T = c.T
    n = 512
    c.prior[0] = (T, F(10000.0), (9, 9, 9, 9))       # saturated; a last record that does not keep stops the rest
    c.run(0, np.r_[np.full(n - 1, 0.5, F), F(0.1)], 1.0)
    c.prior[1] = (T, F(100.0), (1, 1, 1, 1))         # integer weights: warp scan
    c.run(1, np.full(n, 0.5, F), np.random.default_rng(4).integers(1, 6, n).astype(F))
    c.prior[2] = (T, F(1.5), (1, 1, 1, 1))           # non-integer weights: prefix sum
    c.run(2, np.full(n, 0.7, F), F(0.3))
    return c, ["step_saturated", "step_int_scan", "step_prefix"]


def _with_breaks(n, sdf, w):
    """n free-space records whose every 128th (chunk 3, lane 31 of each step) is (sdf 0, weight 0): it fails the
    step's free-space check but leaves a voxel at (+T, W) with T a power of two unchanged, so the other three
    chunks of each step go through the chunk paths."""
    s = np.full(n, sdf, F)
    ww = np.broadcast_to(np.asarray(w, F), (n,)).copy()
    s[127::128] = 0.0
    ww[127::128] = 0.0
    return s, ww


def case_chunk_paths():
    c = Case(0.25, 10000.0)
    T = c.T
    c.prior[0] = (T, F(10000.0), (5, 5, 5, 5))       # saturated
    c.run(0, *_with_breaks(512, 0.5, 1.0))
    c.prior[1] = (T, F(7.0), (5, 5, 5, 5))           # unit weights on an integer W: constant
    c.run(1, *_with_breaks(512, 0.5, 1.0))
    c.prior[2] = (T, F(1.5), (5, 5, 5, 5))           # non-integer weights: prefix
    c.run(2, *_with_breaks(512, 0.5, 0.3))
    c.prior[3] = (T, F(10000.0 - 300.0), (5, 5, 5, 5))  # the max_weight clamp fires: sequential
    c.run(3, *_with_breaks(512, 0.5, 1.0))
    c.prior[4] = (T, F(5e-7), (5, 5, 5, 5))          # W below 1e-6: sequential
    c.run(4, *_with_breaks(256, 0.5, 1.0))
    return c, ["chunk_saturated", "chunk_const", "chunk_prefix", "chunk_sequential", "chunk_exact"]


def case_weight_chain_bounds():
    """Integer weight chains at the float bounds: unit weights from W = 2^22 - 40, 2^22 + 8 and 2^24 - 40 (the
    constant-weight chunk path holds only below 2^22; at 2^24 in-order addition stalls), and integer weights
    2..1000 from 2^24 - 300 (the warp scan holds only while W + sum < 2^24)."""
    c = Case(0.25, 1e30)
    T = c.T
    rng = np.random.default_rng(5)
    for v, W in enumerate((2.0 ** 22 - 40, 2.0 ** 22 + 8, 2.0 ** 24 - 40)):
        c.prior[v] = (T, F(W), (1, 2, 3, 4))
        c.run(v, *_with_breaks(640, 0.5, 1.0))       # chunk paths
        c.prior[8 + v] = (T, F(W), (1, 2, 3, 4))
        c.run(8 + v, np.full(640, 0.5, F), 1.0)      # step paths
    c.prior[4] = (T, F(2.0 ** 24 - 300), (1, 2, 3, 4))
    c.run(4, np.full(1024, 0.5, F), rng.integers(2, 1001, 1024).astype(F))
    c.prior[5] = (T, F(2.0 ** 24 - 300), (1, 2, 3, 4))
    c.run(5, *_with_breaks(1024, 0.5, rng.integers(2, 1001, 1024).astype(F)))
    return c, ["chunk_const", "chunk_prefix", "step_int_scan", "step_prefix"]


def case_step_redone():
    """One record with sdf < T at each of the 128 positions of a step (one voxel per position): the step check
    fails and the step is redone chunk by chunk from the unchanged voxel."""
    c = Case(0.3, 10000.0)
    T = c.T
    rng = np.random.default_rng(6)
    for p in range(128):
        c.prior[p] = (T, F(rng.integers(1, 100)), (7, 7, 7, 7))
        s = np.full(256, 0.9, F)
        s[p] = F(0.05)
        c.run(p, s, rng.choice(np.array([1.0, 2.0, 0.7], F), 256))
    return c, ["chunk_exact", "chunk_prefix", "step_prefix"]


def case_keeps_T_rounding():
    """A free-space run on a voxel at +T whose last record has sdf exactly T (T = 0.3, not exact in binary), at
    each position p of the run's second step: whether (T w + T W) / (W + w) rounds below T depends on the exact
    weight W before the record, so the step's per-lane check -- for every chunk and lane, on integer and on
    non-integer weight chains -- decides the final distance."""
    c = Case(0.3, 1e30)
    T = c.T
    rng = np.random.default_rng(7)
    for v in range(1024):
        p = v % 128
        c.prior[v] = (T, F(rng.integers(1, 300)), (3, 3, 3, 3))
        n = 128 + p + 1
        s = np.full(n, 0.9, F)
        s[-1] = T
        w = rng.integers(1, 9, n).astype(F) if v < 512 else rng.uniform(0.1, 3.0, n).astype(F)
        c.run(v, s, w)
    return c, ["step_int_scan", "step_prefix", "chunk_exact"]


# -- rest at (+T, max_weight) and the keep suffix
def case_rest():
    """Voxels that reach (+T, max_weight) mid-run.  Either every later record keeps (the rest of the run is
    skipped) or one late record does not: in the last record, in the first record of the suffix, in the keep
    word of the rest point, 31, 32 or 33 keep words before the run's end.  Runs start and end off the 32-record
    grid (the voxels before them take 5 records each)."""
    c = Case(0.25, 1000.0)
    T = c.T
    n = 40 * 32 + 13
    rest_at = 100      # W = max_weight - 100 with unit weights: at rest after 100 records
    bad_positions = [None, n - 1, 128, 100, 96, n - 31 * 32, n - 32 * 32, n - 33 * 32, n - 32 * 32 - 17]
    v = 0
    for bad in bad_positions:
        c.prior[v] = (F(0.1), F(3.0), (0, 0, 0, 0))
        c.run(v, np.full(5, 0.1, F), 1.0)                          # shifts the next run off the grid
        v += 1
        c.prior[v] = (T, F(1000.0 - rest_at), (1, 1, 1, 1))
        s = np.full(n, 0.5, F)
        if bad is not None:
            s[bad] = F(0.2)
        c.run(v, s, 1.0)
        v += 1
    return c, ["long_runs", "long_rested", "chunk_sequential"]


# -- edge values of sdf, weight and the prior voxel
def case_sdf_edges():
    """sdf equal to T, nextafter(T, +-inf), -T, 0, and NaN with weight 0 on an observed voxel (what an all-zero-
    weight Merged bundle does: the reference writes -T), in short and long runs."""
    c = Case(0.3, 10000.0)
    T = c.T
    edges = np.array([T, np.nextafter(T, F(np.inf)), np.nextafter(T, F(-np.inf)), -T, 0.0, np.nan], F)
    v = 0
    for n in (1, 3, 40, 200):
        for k, e in enumerate(edges):
            c.prior[v] = (F(0.1 * (k - 2)), F(1.0 + k), (40, 50, 60, 70))
            s = np.full(n, e, F)
            w = np.full(n, 0.0 if np.isnan(e) else 1.0, F)
            c.run(v, s, w)
            v += 1
            c.prior[v] = (T, F(10000.0), (40, 50, 60, 70))              # at rest
            c.run(v, s, w)
            v += 1
    return c, ["short_runs", "long_runs"]


def case_weight_edges():
    """Weights 0, 5e-7 (on an empty voxel: nothing changes), 1e11, and weights that make W + w land exactly on
    max_weight."""
    c = Case(0.3, 10000.0)
    T = c.T
    rng = np.random.default_rng(8)
    v = 0
    for n in (1, 5, 33, 300):
        for w in (0.0, 5e-7, 1e11):
            c.run(v, rng.uniform(-0.5, 0.5, n), w)                       # empty voxel
            v += 1
            c.prior[v] = (F(0.2), F(3.0), (9, 8, 7, 6))
            c.run(v, rng.uniform(-0.5, 0.5, n), w)
            v += 1
        c.prior[v] = (T, F(10000.0 - 0.5 * n), (1, 1, 1, 1))             # lands exactly on max_weight
        c.run(v, np.full(n, 0.5, F), 0.5)
        v += 1
        c.prior[v] = (F(0.1), F(10000.0 - 2.0), (1, 1, 1, 1))
        c.run(v, rng.uniform(-0.5, 0.5, n), 2.0)
        v += 1
    return c, ["short_runs", "long_runs"]


def case_max_weight(max_weight, T):
    """One max_weight against every prior state the reference can meet (a map loaded from a file, pushed through
    setLayer or saved under another max_weight or truncation): (T, mw), (T, 2 mw), (-T, mw), (3T, w), (-0.0, w),
    a weight below 1e-6; each takes free-space runs and mixed runs of many lengths."""
    c = Case(T, max_weight, n_blocks=2)
    T, mw = c.T, c.max_weight
    rng = np.random.default_rng(int(max_weight * 7 + T * 100) % 2 ** 31)
    priors = [(T, mw), (T, F(2) * mw), (-T, mw), (F(3) * T, F(2.5)), (F(-0.0), F(4.0)), (T, F(5e-7)),
              (F(0.0), F(0.0)), (T, F(1.0))]
    v = 0
    for n in (1, 7, 32, 33, 100, 129, 700):
        for d, w in priors:
            for kind in range(3):
                c.prior[v] = (d, w, (rng.integers(0, 256), 7, 99, 255))
                if kind == 0:     # free space, unit weights
                    s, ww = np.full(n, 2 * T, F), np.ones(n, F)
                elif kind == 1:   # free space, non-integer weights
                    s, ww = rng.uniform(T, 3 * T, n).astype(F), rng.uniform(0.0, 2.0, n).astype(F)
                else:             # anything
                    s = rng.uniform(-2 * T, 3 * T, n).astype(F)
                    ww = rng.choice(np.array([0.0, 5e-7, 0.5, 1.0, 3.0, 1e3], F), n)
                c.run(v, s, ww)
                v += 1
    return c, ["long_runs", "short_runs"]


CASES = {
    "run_lengths": case_run_lengths,
    "tile_offsets": case_tile_offsets,
    "runs_of_33_fill_the_pass": case_runs_of_33_fill_the_pass,
    "step_paths": case_step_paths,
    "chunk_paths": case_chunk_paths,
    "weight_chain_bounds": case_weight_chain_bounds,
    "step_redone": case_step_redone,
    "keeps_T_rounding": case_keeps_T_rounding,
    "rest": case_rest,
    "sdf_edges": case_sdf_edges,
    "weight_edges": case_weight_edges,
}
for _mw in (1e-7, 1.0, 5.0, 10000.0, 1e30):
    for _T in (0.25, 0.3):
        CASES[f"max_weight_{_mw:g}_trunc_{_T}"] = (lambda mw=_mw, T=_T: case_max_weight(mw, T))


def _run_case(name):
    out = CASES[name]()
    case, want = out[0], out[1]
    max_updates = out[2] if len(out) > 2 else 0
    paths, ref = check_case(case, max_updates)
    zero = ["long_rested"] if case.max_weight < EPS else []
    _expect(name, paths, want, zero)
    return paths, ref


@pytest.mark.parametrize("name", list(CASES))
def test_apply_against_sequential_reference(name):
    paths, ref = _run_case(name)
    if name == "keeps_T_rounding":
        # the case is sharp: some records do round below T, so a step check that missed one would be seen
        below = ref["distance"][:1024] < F(0.3)
        print("voxels left below T:", int(below[:512].sum()), "(integer weights)", int(below[512:].sum()), "(other)")
        assert below[:512].sum() > 20 and below[512:].sum() > 20
    if name == "rest":
        # the voxels with a late non-keeping record must not rest past it
        assert paths["long_rested"] >= 1


def test_every_path_ran():
    for name in CASES:
        if name not in RAN:
            _run_case(name)
    total = {k: sum(p[k] for p in RAN.values()) for k in PATHS}
    print("all cases:", total)
    assert all(v > 0 for v in total.values()), total


def test_hook_rejects_bad_input():
    layer, integ, idx = _layer(0.3, 100.0, 2, max_updates=1000)
    layer.insertBlocks(idx, np.zeros((2, NV), vb.api.TSDF_DTYPE))
    one = dict(sdf=np.zeros(1, F), w=np.ones(1, F), rgba=np.zeros((1, 4), np.uint8))
    debug_apply(layer, idx, [1], [NV - 1], **one)                              # fine
    with pytest.raises(vb.VoxbloxError):
        debug_apply(layer, idx, [0], [NV], **one)                               # voxel index >= vps^3
    with pytest.raises(vb.VoxbloxError):
        debug_apply(layer, idx, [2], [0], **one)                                # block ordinal out of range
    with pytest.raises(vb.VoxbloxError):
        debug_apply(layer, np.array([[5, 5, 5]], np.int32), [0], [0], **one)   # block not in the map
    with pytest.raises(vb.VoxbloxError):
        debug_apply(layer, np.r_[idx, idx[:1]], [0], [0], **one)               # a block listed twice
    n = 1001
    with pytest.raises(vb.VoxbloxError):
        debug_apply(layer, idx, np.zeros(n), np.zeros(n), np.zeros(n, F), np.ones(n, F), np.zeros((n, 4), np.uint8))
    # the map still works afterwards
    debug_apply(layer, idx, [0, 0], [3, 3], np.array([0.1, 0.2], F), np.ones(2, F), np.zeros((2, 4), np.uint8))
    vox, _ = layer.getBlocks(idx)
    assert vox["weight"].reshape(-1)[3] == 2.0


def test_hook_voxels_per_side_8():
    """The apply with 512-voxel blocks (record keys carry 9 voxel bits)."""
    n_vox = 8 ** 3
    cfg = vb.TsdfIntegratorConfig(default_truncation_distance=0.3, max_weight=50.0, integrator_threads=1)
    layer = vb.Layer(0.1, 8)
    vb.TsdfIntegratorFactory.create("simple", cfg, layer)
    idx = np.array([[0, 0, 0], [-1, 2, 3], [7, -4, 0]], np.int32)
    rng = np.random.default_rng(9)
    prior = np.zeros(3 * n_vox, vb.api.TSDF_DTYPE)
    prior["distance"] = rng.uniform(-0.3, 0.3, prior.size).astype(F)
    prior["weight"] = rng.choice(np.array([0.0, 1.0, 50.0, 100.0], F), prior.size)
    layer.insertBlocks(idx, prior.reshape(3, n_vox))
    n = 50000
    vox = rng.integers(0, 3 * n_vox, n)
    vox[:5000] = 17          # one long run
    sdf = rng.uniform(-0.6, 0.9, n).astype(F)
    w = rng.uniform(0.0, 3.0, n).astype(F)
    rgba = rng.integers(0, 256, (n, 4)).astype(np.uint8)
    paths = debug_apply(layer, idx, vox // n_vox, vox % n_vox, sdf, w, rgba)
    ref = prior.copy()
    reference_apply(ref, vox, sdf, w, rgba, 0.3, 50.0)
    got, _ = layer.getBlocks(idx)
    assert got.reshape(-1).tobytes() == ref.tobytes()
    assert paths["long_runs"] > 0 and paths["short_runs"] > 0, paths
