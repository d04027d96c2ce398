"""-m gpu: ICP's per-batch arithmetic run on the device (vbx_debug_icp_solve: the functions of
voxblox_b200/csrc/vbx_icp_math.cuh that k_icp applies to each mini batch) against the same header built for
the host (tests/icp_math_check.cc), on the families of tests/test_icp_math_cpu.py.  The algebraic parts (the
Procrustes solve, its validity decision and the quaternion of a matrix) must be bit identical; log and exp call
the platform's acos / asin / sin / cos, which may differ between CUDA and the host's libm: CUDA's asinf / acosf
are within 2 ulp, and log divides and multiplies their result twice more (4 ulp allowed); exp rounds a double
result to float (2 ulp allowed)."""
import ctypes as C

import numpy as np
import pytest

import voxblox_b200 as vb
from tests import test_icp_math_cpu as hm

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    layer = vb.Layer(0.1, 16)
    vb.TsdfIntegratorFactory.create("merged", vb.TsdfIntegratorConfig(), layer)
    return layer._ctx


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    return hm.build(str(tmp_path_factory.mktemp("icp_math")))[0]


def device_batch(ctx, h, m, q, w, refine_roll_pitch):
    n = len(h)
    h, m, q, w = (np.ascontiguousarray(a, np.float32) for a in (h, m, q, w))
    r = np.zeros((n, 3, 3), np.float32)
    valid = np.zeros(n, np.int32)
    qo = np.zeros((n, 4), np.float32)
    lo = np.zeros((n, 3), np.float32)
    eo = np.zeros((n, 4), np.float32)
    ctx.check(ctx.lib.vbx_debug_icp_solve(ctx.handle, C.c_uint32(n), C.c_int(refine_roll_pitch), h.ctypes.data,
                                          m.ctypes.data, q.ctypes.data, w.ctypes.data, r.ctypes.data, valid.ctypes.data,
                                          qo.ctypes.data, lo.ctypes.data, eo.ctypes.data), "vbx_debug_icp_solve")
    return r, valid, qo, lo, eo


def _ulps(a, b):
    """distance in float32 steps (same-sign floats; 0 and -0 are 0 apart)"""
    ia = a.astype(np.float32).view(np.int32).astype(np.int64)
    ib = b.astype(np.float32).view(np.int32).astype(np.int64)
    ia = np.where(ia < 0, np.int64(-(2 ** 31)) - ia, ia)
    ib = np.where(ib < 0, np.int64(-(2 ** 31)) - ib, ib)
    return np.abs(ia - ib)


def _inputs():
    """Every family's H, next to the quaternion-branch matrices and the log / exp inputs (cycled to the same length)."""
    h = np.concatenate([hm.family(name, n=500) for name in hm.FAMILIES])
    n = len(h)
    m = hm.quat_inputs()
    q, w = hm.log_exp_inputs()
    take = lambda a: a[np.arange(n) % len(a)]
    return h, take(m), take(q), take(w)


@pytest.mark.parametrize("refine_roll_pitch", [0, 1])
def test_device_per_batch_math_equals_the_host_build(ctx, host, refine_roll_pitch):
    h, m, q, w = _inputs()
    dev = device_batch(ctx, h, m, q, w, refine_roll_pitch)
    ref = hm.math_batch(host, h, m, q, w, refine_roll_pitch)
    for name, d, r in zip(("rotation", "valid", "quat_from_matrix"), dev[:3], ref[:3]):
        bad = np.flatnonzero((d.view(np.uint32) != r.view(np.uint32)).reshape(len(h), -1).any(axis=1))
        assert bad.size == 0, (name, bad[:10], d[bad[:1]], r[bad[:1]])
    assert ref[1].all()
    for name, d, r, bound in zip(("log", "exp"), dev[3:], ref[3:], (4, 2)):
        u = _ulps(d, r)
        print(name, "max ulp", int(u.max()))
        assert u.max() <= bound, (name, int(u.max()), int(u.argmax()))
