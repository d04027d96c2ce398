"""ICP's per-batch arithmetic (voxblox_b200/csrc/vbx_icp_math.cuh, built for the host by tests/icp_math_check.cc)
against float64 references: numpy's SVD and Kabsch solution for the Procrustes rotation, scipy's Rotation for
the quaternion of a matrix, the closed forms of minkindr's SO(3) log / exp, and the float64 form of one fusion
step (icp.cc:195-213).  The mini batches are 20 float points, as ICP's default mini_batch_size makes them,
in seeded families that reach every branch: random, planar (rank-2 H), collinear (rank 1), H = 0, det H < 0,
repeated singular values, optimum rotations near pi, and H scaled from 1e-6 to 1e4.

Also the test build's stand-in JacobiSVD (oracle/shim/Eigen/Core, which the reference library is compiled
against; tests/shim_svd_check.cc) against its own contract: U and V orthonormal, H = U S V^T, S decreasing."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
from scipy.spatial.transform import Rotation

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
N_BATCH = 2000   # batches per family
FAMILIES = ["random", "planar", "collinear", "zero", "negative_det", "repeated", "near_pi_x", "near_pi_y",
            "near_pi_z", "scaled"]
F32 = np.float32


def build(tmp_dir):
    """The host harness (the product header) and the shim driver, built into tmp_dir."""
    ic = os.path.join(tmp_dir, "libicp_math_check.so")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-x", "c++",
                           os.path.join(HERE, "icp_math_check.cc"), "-o", ic])
    sh = os.path.join(tmp_dir, "libshim_svd_check.so")
    subprocess.check_call(["g++", "-std=c++14", "-O2", "-ffp-contract=off", "-fPIC", "-shared",
                           "-I", os.path.join(ROOT, "oracle", "shim"), os.path.join(HERE, "shim_svd_check.cc"), "-o", sh])
    return C.CDLL(ic), C.CDLL(sh)


@pytest.fixture(scope="module")
def libs(tmp_path_factory):
    return build(str(tmp_path_factory.mktemp("icp_math")))


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def math_batch(lib, h, m, q, w, refine_roll_pitch):
    """icp_math_batch over n items: (r [n,3,3], valid [n], quat of m [n,4], log q [n,3], exp w [n,4])."""
    n = len(h)
    h, m, q, w = (np.ascontiguousarray(a, F32) for a in (h, m, q, w))
    r = np.zeros((n, 3, 3), F32)
    valid = np.zeros(n, np.int32)
    qo = np.zeros((n, 4), F32)
    lo = np.zeros((n, 3), F32)
    eo = np.zeros((n, 4), F32)
    lib.icp_math_batch(C.c_uint32(n), C.c_int(refine_roll_pitch), _ptr(h), _ptr(m), _ptr(q), _ptr(w), _ptr(r),
                       _ptr(valid), _ptr(qo), _ptr(lo), _ptr(eo))
    return r, valid, qo, lo, eo


def _rotations(rng, n, angle=None, axis=None):
    """n random rotations (float64 matrices); `angle` (low, high) and `axis` (a unit vector, jittered) restrict them."""
    if angle is None:
        return Rotation.random(n, random_state=rng).as_matrix()
    ax = rng.normal(size=(n, 3)) if axis is None else np.asarray(axis, float) + 0.15 * rng.normal(size=(n, 3))
    ax /= np.linalg.norm(ax, axis=1, keepdims=True)
    return Rotation.from_rotvec(ax * rng.uniform(*angle, size=(n, 1))).as_matrix()


def _cross_cov(src, tgt):
    """H = sum_k (src_k - mean) (tgt_k - mean)^T in float32, summed point by point as ICP does (icp.h:156-157)."""
    src, tgt = src.astype(F32), tgt.astype(F32)
    sd = src - src.mean(axis=1, keepdims=True, dtype=F32)
    td = tgt - tgt.mean(axis=1, keepdims=True, dtype=F32)
    h = np.zeros((src.shape[0], 3, 3), F32)
    for k in range(src.shape[1]):
        h += sd[:, k, :, None] * td[:, k, None, :]
    return h


def family(name, n=N_BATCH, seed=0):
    """n float32 cross-covariances H of 20-point mini batches."""
    rng = np.random.default_rng([FAMILIES.index(name), seed])
    rot = _rotations(rng, n)
    if name == "zero":
        return np.zeros((n, 3, 3), F32)
    if name == "repeated":   # H = U diag(s) V^T with two equal singular values, either pair, either det sign
        u, v = _rotations(rng, n), _rotations(rng, n)
        s = np.ones((n, 3))
        s[: n // 2, 2] = rng.uniform(0.01, 0.9, n // 2)
        s[n // 2:, 0] = rng.uniform(1.1, 100, n - n // 2)
        s[::3, 2] *= -1.0
        return np.einsum("nij,nj,nkj->nik", u, s, v).astype(F32)
    src = rng.normal(size=(n, 20, 3)) * rng.uniform(0.2, 3.0, size=(n, 1, 3))
    if name == "planar":
        src[:, :, 2] = 0.0
        src = np.einsum("nij,nkj->nki", rot, src)
    elif name == "collinear":
        src = rng.normal(size=(n, 20, 1)) * rng.normal(size=(n, 1, 3))
    if name.startswith("near_pi"):   # optimum rotations of 2.2 .. pi rad: trace(R) <= 0, quat_from_matrix's i = 0, 1, 2
        axis = np.eye(3)["xyz".index(name[-1])]
        rot = _rotations(rng, n, angle=(2.2, np.pi), axis=axis)
    if name == "negative_det":   # the target mirrored: the optimum proper rotation has det(V U^T) flipped
        rot = rot * np.array([1.0, 1.0, -1.0])
    tgt = np.einsum("nij,nkj->nki", rot, src) + rng.uniform(0.0, 0.05, size=(n, 1, 1)) * rng.normal(size=src.shape)
    h = _cross_cov(src, tgt)
    if name == "scaled":
        h = (h * 10.0 ** rng.uniform(-6.0, 4.0, size=(n, 1, 1))).astype(F32)
    return h


# ---------------------------------------------------------------------------------------------- float64 references
def kabsch(h, dim):
    """The proper rotation maximising trace(R H) in float64 (top-left dim x dim block of H), its optimum value and
    whether the optimum is unique (then R is compared): sigma_2 > 1e-3 sigma_1, and for det H < 0 also
    sigma_2 - sigma_3 > 1e-3 sigma_1 (else a one-parameter family ties)."""
    hd = h[:, :dim, :dim].astype(np.float64)
    u, s, vt = np.linalg.svd(hd)
    d = np.sign(np.linalg.det(u) * np.linalg.det(vt))
    d[d == 0] = 1.0
    dd = np.ones((len(h), dim))
    dd[:, -1] = d
    r = np.einsum("nji,nj,nkj->nik", vt, dd, u)   # V diag(1, .., d) U^T
    best = (s * dd).sum(axis=1)
    sig = np.linalg.svd(hd, compute_uv=False)
    unique = sig[:, 1] > 1e-3 * sig[:, 0]
    neg = np.linalg.det(hd) < 0
    unique &= ~neg | (sig[:, dim - 2] - sig[:, dim - 1] > 1e-3 * sig[:, 0])
    return r, best, unique


def _rotation_report(r, h, dim):
    r64 = r.astype(np.float64)
    orth = np.abs(np.einsum("nij,nkj->nik", r64, r64) - np.eye(3)).max(axis=(1, 2))
    det = np.abs(np.linalg.det(r64) - 1.0)
    rk, best, unique = kabsch(h, dim)
    got = np.einsum("nij,nji->n", r64[:, :dim, :dim], h[:, :dim, :dim].astype(np.float64))
    short = (best - got) / np.maximum(np.abs(best), 1e-300)   # relative loss in trace(R H)
    err = np.abs(r64[:, :dim, :dim] - rk).max(axis=(1, 2))
    return orth, det, short, err, unique


@pytest.mark.parametrize("name", FAMILIES)
def test_3d_rotation_is_the_procrustes_optimum(libs, name):
    h = family(name)
    n = len(h)
    r, valid, *_ = math_batch(libs[0], h, np.tile(np.eye(3), (n, 1, 1)), np.tile([1, 0, 0, 0], (n, 1)),
                              np.zeros((n, 3)), 1)
    orth, det, short, err, unique = _rotation_report(r, h, 3)
    rep = dict(orth=orth.max(), det=det.max(), short=short.max(), err=err[unique].max(initial=0.0),
               n_unique=int(unique.sum()), invalid=int((valid == 0).sum()))
    assert orth.max() <= 1e-5 and det.max() <= 1e-5, rep
    assert short.max() <= 1e-5, rep
    assert err[unique].max(initial=0.0) <= 1e-5, rep
    assert valid.all(), rep                       # ICP fuses every one of them, as voxblox on Eigen does
    if name in ("random", "near_pi_x", "scaled", "negative_det"):
        assert unique.mean() > 0.9, rep           # the comparison with Kabsch is not vacuous
    if name == "zero":
        assert (r == np.eye(3, dtype=F32)).all()


@pytest.mark.parametrize("name", FAMILIES)
def test_2d_rotation_is_the_procrustes_optimum(libs, name):
    h = family(name)
    n = len(h)
    r, valid, *_ = math_batch(libs[0], h, np.tile(np.eye(3), (n, 1, 1)), np.tile([1, 0, 0, 0], (n, 1)),
                              np.zeros((n, 3)), 0)
    orth, det, short, err, unique = _rotation_report(r, h, 2)
    rep = dict(orth=orth.max(), det=det.max(), short=short.max(), err=err[unique].max(initial=0.0),
               invalid=int((valid == 0).sum()))
    assert orth.max() <= 1e-5 and det.max() <= 1e-5, rep
    assert short.max() <= 1e-5, rep
    assert err[unique].max(initial=0.0) <= 1e-5, rep
    assert valid.all(), rep
    assert (r[:, 2] == [0, 0, 1]).all() and (r[:, :, 2] == [0, 0, 1]).all()
    if name == "zero":   # H = 0: the SVD's U = V = I, a translation-only step
        assert (r == np.eye(3, dtype=F32)).all()


# ----------------------------------------------------------------------------------------- quaternion conversions
def quat_inputs(seed=0):
    """Rotation matrices reaching every branch of quat_from_matrix: trace > 0, and trace <= 0 with the largest
    diagonal entry at 0, 1 and 2; the identity and exact half turns about the axes."""
    rng = np.random.default_rng([77, seed])
    parts = [_rotations(rng, 500), _rotations(rng, 300, angle=(0.0, 0.3))]
    for axis in np.eye(3):
        parts.append(_rotations(rng, 300, angle=(2.2, np.pi), axis=axis))
    parts.append(np.stack([np.eye(3), np.diag([1.0, -1, -1]), np.diag([-1.0, 1, -1]), np.diag([-1.0, -1, 1])]))
    return np.concatenate(parts).astype(F32)


def test_quat_from_matrix_matches_scipy_on_every_branch(libs):
    m = quat_inputs()
    n = len(m)
    tr = np.trace(m.astype(np.float64), axis1=1, axis2=2)
    big = np.argmax(np.diagonal(m, axis1=1, axis2=2), axis=1)
    assert (tr > 0).sum() > 100 and all(((tr <= 0) & (big == i)).sum() > 100 for i in range(3))
    _, _, q, _, _ = math_batch(libs[0], np.zeros((n, 3, 3)), m, np.tile([1, 0, 0, 0], (n, 1)), np.zeros((n, 3)), 1)
    ref = Rotation.from_matrix(m.astype(np.float64)).as_quat()[:, [3, 0, 1, 2]]   # (w, x, y, z)
    err = np.minimum(np.abs(q - ref).max(axis=1), np.abs(q + ref).max(axis=1))
    assert err.max() <= 1e-6, (err.max(), int(err.argmax()))


def log_exp_inputs(seed=0):
    """Quaternions for log and rotation vectors for exp whose angles cross both series thresholds (float
    eps^(1/4) ~ 0.0186 on |vec(q)| in log, double eps^(1/4) ~ 1.2e-4 on the angle in exp), reach pi, and, for
    log, quaternions with negative w (eta < 0)."""
    rng = np.random.default_rng([91, seed])
    e4f, e4d = float(np.finfo(F32).eps) ** 0.25, float(np.finfo(np.float64).eps) ** 0.25
    half = np.concatenate([10.0 ** rng.uniform(-8, -1, 400), np.arcsin(e4f) * (1 + rng.uniform(-1e-3, 1e-3, 200)),
                           rng.uniform(0.0, np.pi / 2, 400), np.pi / 2 - 10.0 ** rng.uniform(-7, -1, 100), [0.0, np.pi / 2]])
    ax = rng.normal(size=(len(half), 3))
    ax /= np.linalg.norm(ax, axis=1, keepdims=True)
    q = np.concatenate([np.cos(half)[:, None], np.sin(half)[:, None] * ax], axis=1)
    q[::2] *= -1.0                                                   # eta < 0: the same rotation
    theta = np.concatenate([10.0 ** rng.uniform(-9, -3, 400), e4d * (1 + rng.uniform(-1e-3, 1e-3, 200)),
                            rng.uniform(0.0, np.pi, 400), np.pi - 10.0 ** rng.uniform(-7, -1, 100), [0.0, np.pi]])
    ax = rng.normal(size=(len(theta), 3))
    ax /= np.linalg.norm(ax, axis=1, keepdims=True)
    return q.astype(F32), (theta[:, None] * ax).astype(F32)


def log_ref(q):
    """minkindr RotationQuaternion::log on the float32 input, in float64 and without the series."""
    q = q.astype(np.float64)
    eta, a = q[:, 0], q[:, 1:]
    na = np.linalg.norm(a, axis=1)
    with np.errstate(divide="ignore", invalid="ignore"):
        acos_branch = np.where(eta >= 0, np.arccos(np.clip(eta, -1, 1)), -np.arccos(np.clip(-eta, -1, 1))) / na
        asin_branch = np.where(na > 0, np.arcsin(np.minimum(na, 1.0)) / na, 1.0) * np.where(eta > 0, 1.0, -1.0)
    scale = np.where(np.abs(eta) < na, acos_branch, asin_branch)
    return a * (2.0 * scale)[:, None]


def exp_ref(w):
    w = w.astype(np.float64)
    th = np.linalg.norm(w, axis=1)
    with np.errstate(divide="ignore", invalid="ignore"):
        s = np.where(th > 0, np.sin(th / 2) / th, 0.5)
    return np.concatenate([np.cos(th / 2)[:, None], w * s[:, None]], axis=1)


def ulp_error(got, ref):
    """|got - ref| in units of the float32 spacing at |ref| (per coefficient; the largest coefficient's spacing
    for coefficients far below it, whose absolute error follows the shared scale)."""
    big = np.abs(ref).max(axis=1, keepdims=True)
    unit = np.spacing(np.maximum(np.abs(ref), big * 2.0 ** -8).astype(F32)).astype(np.float64)
    return np.abs(got.astype(np.float64) - ref) / np.where(unit > 0, unit, np.spacing(F32(0)))


def test_log_and_exp_match_float64_across_their_series_thresholds(libs):
    q, w = log_exp_inputs()
    n = max(len(q), len(w))
    q = np.concatenate([q, np.tile(q[:1], (n - len(q), 1))])
    w = np.concatenate([w, np.tile(w[:1], (n - len(w), 1))])
    _, _, _, lg, ex = math_batch(libs[0], np.zeros((n, 3, 3)), np.tile(np.eye(3), (n, 1, 1)), q, w, 1)
    el, ee = ulp_error(lg, log_ref(q)), ulp_error(ex, exp_ref(w))
    assert el.max() <= 4, (el.max(), q[int(el.max(axis=1).argmax())])
    assert ee.max() <= 1, (ee.max(), w[int(ee.max(axis=1).argmax())])


# -------------------------------------------------------------------------------------------------- one fusion step
def _qmul(a, b):
    w1, x1, y1, z1 = a.T
    w2, x2, y2, z2 = b.T
    return np.stack([w1 * w2 - x1 * x2 - y1 * y2 - z1 * z2, w1 * x2 + x1 * w2 + y1 * z2 - z1 * y2,
                     w1 * y2 + y1 * w2 + z1 * x2 - x1 * z2, w1 * z2 + z1 * w2 + x1 * y2 - y1 * x2], axis=1)


def _qrot(q, p):
    qv = q[:, 1:]
    uv = 2.0 * np.cross(qv, p)
    return p + q[:, :1] * uv + np.cross(qv, uv)


def fuse_ref(cur, base, delta, info):
    """icp.cc:195-213 in float64: d = cur^-1 (delta cur); cur <- cur exp(w .* log d), w = info / (base + info)."""
    cq, ct, dq, dt = cur[:, :4], cur[:, 4:], delta[:, :4], delta[:, 4:]
    tq, tt = _qmul(dq, cq), dt + _qrot(dq, ct)                     # t_temp = delta * cur
    ci = cq * np.array([1.0, -1, -1, -1])
    lq, lt = _qmul(ci, tq), _qrot(ci, tt - ct)                     # cur^-1 * t_temp
    lg = np.concatenate([lt, log_ref(lq)], axis=1)
    wl = info / (base + info) * lg
    eq = exp_ref(wl[:, 3:])
    return np.concatenate([_qmul(cq, eq), ct + _qrot(cq, wl[:, :3])], axis=1), base + info


def test_one_fusion_step_matches_float64(libs):
    rng = np.random.default_rng(5)
    n = 3000
    cq = Rotation.random(n, random_state=rng).as_quat()[:, [3, 0, 1, 2]]
    cur = np.concatenate([cq, rng.normal(size=(n, 3)) * 3.0], axis=1).astype(F32)
    small = rng.uniform(size=(n, 1)) < 0.7   # ICP's steps are small; large ones (up to pi) as well
    ang = np.where(small, 10.0 ** rng.uniform(-7, -1, (n, 1)), rng.uniform(0, np.pi, (n, 1)))
    ax = rng.normal(size=(n, 3))
    ax /= np.linalg.norm(ax, axis=1, keepdims=True)
    dq = np.concatenate([np.cos(ang / 2), np.sin(ang / 2) * ax], axis=1)
    delta = np.concatenate([dq, rng.normal(size=(n, 3)) * np.where(small, 0.01, 1.0)], axis=1).astype(F32)
    base = (10.0 ** rng.uniform(0, 4, (n, 6))).astype(F32)
    info = (10.0 ** rng.uniform(-2, 3, (n, 6))).astype(F32)
    got, gbase = cur.copy(), base.copy()
    libs[0].icp_fuse_batch(C.c_uint32(n), _ptr(got), _ptr(gbase), _ptr(delta), _ptr(info))
    ref, rbase = fuse_ref(cur.astype(np.float64), base.astype(np.float64), delta.astype(np.float64),
                          info.astype(np.float64))
    assert np.abs(gbase - rbase).max() <= np.spacing(rbase.astype(F32)).max()
    dq_err = np.abs(got[:, :4] - ref[:, :4]).max(axis=1)
    dt_err = np.abs(got[:, 4:] - ref[:, 4:]).max(axis=1) / np.maximum(1.0, np.abs(ref[:, 4:]).max(axis=1))
    assert dq_err.max() <= 2e-6 and dt_err.max() <= 2e-6, (dq_err.max(), dt_err.max())


# ------------------------------------------------------------------------------------ the reference build's SVD
@pytest.mark.parametrize("dim", [2, 3])
@pytest.mark.parametrize("name", FAMILIES)
def test_shim_jacobi_svd_meets_its_contract(libs, name, dim):
    h = np.ascontiguousarray(family(name)[:, :dim, :dim])
    n = len(h)
    u = np.zeros_like(h)
    v = np.zeros_like(h)
    libs[1].shim_svd(C.c_int(dim), C.c_uint32(n), _ptr(h), _ptr(u), _ptr(v))
    u64, v64, h64 = u.astype(np.float64), v.astype(np.float64), h.astype(np.float64)
    eye = np.eye(dim)
    orth = max(np.abs(np.einsum("nji,njk->nik", u64, u64) - eye).max(), np.abs(np.einsum("nji,njk->nik", v64, v64) - eye).max())
    s = np.einsum("nji,njk,nkl->nil", u64, h64, v64)               # U^T H V
    sig = np.linalg.svd(h64, compute_uv=False)
    scale = np.maximum(sig[:, :1], 1e-300)
    diag = np.diagonal(s, axis1=1, axis2=2)
    off = np.abs(s - np.einsum("ni,ij->nij", diag, eye)).max(axis=(1, 2)) / scale[:, 0]
    rec = np.abs(h64 - np.einsum("nij,nj,nkj->nik", u64, sig, v64)).max(axis=(1, 2)) / scale[:, 0]
    desc = (np.diff(diag, axis=1) / scale).max(initial=-1.0)
    rep = dict(orth=orth, off=off.max(), rec=rec.max(), desc=desc, neg=(diag / scale).min())
    assert orth <= 1e-6, rep
    assert rec.max() <= 1e-5 and off.max() <= 1e-5, rep           # H = U S V^T with S = the singular values
    assert desc <= 1e-5 and (diag / scale).min() >= -1e-5, rep     # S >= 0, decreasing
