"""-m gpu: ICP on clouds whose mini batches are degenerate, on the device against the restatement and (one
thread) against the reference's own voxblox::ICP, whose poses are recorded in tests/golden/reference_pins.json.

  * wall: scenes.c1_planar_wall, a single plane: with refine_roll_pitch every batch's cross-covariance H has
    rank 2, its third singular value rounding noise (~1e-8 of the first);
  * repeated: one surface point 200 times from the identity pose: the demeaned batch is exactly zero, so H = 0
    (2-D) or, once a step has moved the pose, a rank-1 H of rounding residues.

Every such batch must give a proper rotation that ICP fuses (voxblox on Eigen does), and the fused pose a unit
quaternion.  Bounds as in tests/test_icp_gpu.py: 1e-4 on the quaternion, relative to max(1, |t|) on t."""
import numpy as np
import pytest

import voxblox_b200 as vb
from oracle import pyoracle as po
from tests.golden import reference_pins as pins
from tests.test_icp_gpu import TOL, _close, _maps, _perturbed
from voxblox_b200 import scenes

pytestmark = pytest.mark.gpu

VOXEL, TRUNC = 0.2, 0.8
SCENES = ["wall", "repeated"]
PIN_KEYS = [f"{name}/refine_roll_pitch_{r}" for name in SCENES for r in (0, 1)]


def cloud(name):
    """(points, initial q, initial t) of the ICP run on the map of scenes.c1_planar_wall."""
    s = scenes.c1_planar_wall()
    if name == "wall":
        q0, t0 = _perturbed(s, (0.03, -0.02, 0.05), 0.01)
        return s[0], q0, t0
    # a point of the wall at z = 3 whose coordinates are short enough binary fractions that the mean of 20
    # copies is the point itself
    return np.tile(np.array([[0.25, -0.5, 3.0]], np.float32), (200, 1)), np.array([1, 0, 0, 0], np.float32), np.zeros(3, np.float32)


def reference_side(key, lib):
    """The oracle's map of the wall scan and its one-thread ICP of `key`'s cloud: {"map": digest, "icp": {...}}."""
    name, rrp = key.split("/")[0], int(key[-1])
    s = scenes.c1_planar_wall()
    omap = po.OracleMap(lib, po.TsdfConfig(default_truncation_distance=TRUNC, integrator_threads=1), VOXEL, 16)
    omap.integrate(po.MERGED, s)
    pts, q0, t0 = cloud(name)
    q, t, n = omap.icp(po.IcpConfig(refine_roll_pitch=rrp), pts, q0, t0, 11)
    icp = {"q_wxyz": [float(v).hex() for v in q], "t": [float(v).hex() for v in t], "num_updates": int(n)}
    return omap, {"map": pins.map_digest(omap), "icp": icp}


@pytest.fixture(scope="module")
def maps():
    return _maps("port", VOXEL, TRUNC, [scenes.c1_planar_wall()])


def _check(dev, ref):
    rep = _close(dev, ref)
    rep["unit"] = abs(float(np.linalg.norm(dev[1][0].astype(np.float64))) - 1.0)
    assert rep["dq"] <= TOL and rep["dt_rel"] <= TOL, rep
    assert rep["unit"] <= 1e-6, rep
    return rep


@pytest.mark.parametrize("refine_roll_pitch", [0, 1])
@pytest.mark.parametrize("name", SCENES)
def test_degenerate_batches_one_thread_against_the_reference(maps, name, refine_roll_pitch):
    key = f"{name}/refine_roll_pitch_{refine_roll_pitch}"
    _, got = reference_side(key, pins.lib())
    want = pins.recorded(f"icp_degenerate/{key}")
    assert got["map"] == want["map"], "the oracle's map is not the reference's"
    layer, _ = maps
    pts, q0, t0 = cloud(name)
    dev = vb.ICP(vb.ICPConfig(refine_roll_pitch=refine_roll_pitch)).runICP(layer, pts, (q0, t0), seed=11)
    r = want["icp"]
    ref = (np.array([float.fromhex(v) for v in r["q_wxyz"]]), np.array([float.fromhex(v) for v in r["t"]]), r["num_updates"])
    rep = _check(dev, ref)
    print(key, rep)
    assert rep["updates"][0] == rep["updates"][1] > 0, rep


@pytest.mark.parametrize("threads", [1, 4])
@pytest.mark.parametrize("refine_roll_pitch", [0, 1])
@pytest.mark.parametrize("name", SCENES)
def test_degenerate_batches_against_the_restatement(maps, name, refine_roll_pitch, threads):
    layer, omap = maps
    pts, q0, t0 = cloud(name)
    cfg = dict(refine_roll_pitch=refine_roll_pitch, num_threads=threads)
    dev = vb.ICP(vb.ICPConfig(**cfg)).runICP(layer, pts, (q0, t0), seed=11)
    ref = omap.icp(po.IcpConfig(**cfg), pts, q0, t0, 11)
    rep = _check(dev, ref)
    print(name, cfg, rep)
    assert rep["updates"][0] == rep["updates"][1] > 0, rep
