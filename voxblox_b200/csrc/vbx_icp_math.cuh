// The per-batch arithmetic of ICP (vbx_icp.cu): the Procrustes rotation of one mini batch, its validity
// test, the quaternion conversions, minkindr's SO(3) log / exp, the SE(3) products and the fusion of one
// batch's step into the running pose.
//
// Reference: voxblox::ICP::getRotationFromMatchedPoints (include/voxblox/alignment/icp.h:146-190) and the
// fusion of runThread (src/alignment/icp.cc:195-213).  Float32 with one rounding per operation (the
// library is built with -fmad=false), in the operation order of the reference's Eigen / minkindr
// expressions; the 3-D SVD works in double.  The same header compiles for the host (plain IEEE ops; build
// with -ffp-contract=off) so that tests/ can hold it to a float64 reference without a GPU: the algebraic
// functions give the same bits on both sides, log / exp call the platform's libm (asin / acos / sin / cos).
#pragma once

#include <float.h>
#include <math.h>

#include "vbx_math.cuh"

namespace vbx {

struct IcpQuat {
  float w, x, y, z;
};
struct IcpSE3 {
  IcpQuat q;
  F3 t;
};

VBX_HD IcpQuat icp_qmul(const IcpQuat& a, const IcpQuat& b) {
  IcpQuat r;
  r.w = a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z;
  r.x = a.w * b.x + a.x * b.w + a.y * b.z - a.z * b.y;
  r.y = a.w * b.y + a.y * b.w + a.z * b.x - a.x * b.z;
  r.z = a.w * b.z + a.z * b.w + a.x * b.y - a.y * b.x;
  return r;
}
VBX_HD F3 icp_qrot(const IcpQuat& q, F3 p) {
  const F3 qv = f3(q.x, q.y, q.z);
  F3 uv = cross3(qv, p);
  uv = add3(uv, uv);
  return add3(add3(p, scale3(uv, q.w)), cross3(qv, uv));
}
VBX_HD IcpSE3 icp_mul(const IcpSE3& a, const IcpSE3& b) {
  IcpSE3 r;
  r.q = icp_qmul(a.q, b.q);
  r.t = add3(a.t, icp_qrot(a.q, b.t));
  return r;
}
VBX_HD IcpSE3 icp_inv(const IcpSE3& a) {
  IcpSE3 r;
  r.q.w = a.q.w;
  r.q.x = -a.q.x;
  r.q.y = -a.q.y;
  r.q.z = -a.q.z;
  const F3 v = icp_qrot(r.q, a.t);
  r.t = f3(-v.x, -v.y, -v.z);
  return r;
}
// Eigen: quaternion <- rotation matrix
VBX_HD IcpQuat icp_quat_from_matrix(const float m[3][3]) {
  IcpQuat q;
  float t = m[0][0] + m[1][1] + m[2][2];
  if (t > 0.0f) {
    t = sqrtf(t + 1.0f);
    q.w = 0.5f * t;
    t = 0.5f / t;
    q.x = (m[2][1] - m[1][2]) * t;
    q.y = (m[0][2] - m[2][0]) * t;
    q.z = (m[1][0] - m[0][1]) * t;
  } else {
    int i = 0;
    if (m[1][1] > m[0][0]) i = 1;
    if (m[2][2] > m[i][i]) i = 2;
    const int j = (i + 1) % 3, k = (j + 1) % 3;
    float v[3];
    t = sqrtf(m[i][i] - m[j][j] - m[k][k] + 1.0f);
    v[i] = 0.5f * t;
    t = 0.5f / t;
    q.w = (m[k][j] - m[j][k]) * t;
    v[j] = (m[j][i] + m[i][j]) * t;
    v[k] = (m[k][i] + m[i][k]) * t;
    q.x = v[0];
    q.y = v[1];
    q.z = v[2];
  }
  return q;
}
// minkindr RotationQuaternion::log / exp; eps4_f = float epsilon^(1/4), eps4_d = double epsilon^(1/4)
VBX_HD F3 icp_quat_log(const IcpQuat& q, float eps4_f) {
  const F3 a = f3(q.x, q.y, q.z);
  const float na = norm3(a), eta = q.w;
  float scale;
  if (fabsf(eta) < na) {
    scale = eta >= 0.0f ? acosf(eta) / na : -acosf(-eta) / na;
  } else {
    const float s = fabsf(na) < eps4_f ? 1.0f + na * na * (float)(1.0 / 6.0) : asinf(na) / na;
    scale = eta > 0.0f ? s : -s;
  }
  return scale3(a, 2.0f * scale);
}
VBX_HD IcpQuat icp_quat_exp(F3 d, double eps4_d) {
  const double x = d.x, y = d.y, z = d.z;
  const double theta = sqrt(x * x + y * y + z * z);
  const double na = theta < eps4_d ? 0.5 + (theta * theta) * (1.0 / 48.0) : sin(theta * 0.5) / theta;
  IcpQuat q;
  q.w = (float)cos(theta * 0.5);
  q.x = (float)(x * na);
  q.y = (float)(y * na);
  q.z = (float)(z * na);
  return q;
}

// 2-D Procrustes (refine_roll_pitch = false): the proper rotation V diag(1, det) U^T of the 2 x 2 SVD of
// H's top-left block maximises trace(R H) = c (h00 + h11) + s (h01 - h10), so it is the closed form below.
VBX_HD void icp_rotation_2d(const float h[3][3], float r[3][3]) {
  const float a = fadd(h[0][0], h[1][1]), b = fsub(h[0][1], h[1][0]);
  const float nrm = fsqrt(fadd(fmul(a, a), fmul(b, b)));
  // a = b = 0 (H = 0: a batch of repeated points): every rotation is optimal, and the SVD of H = 0 has
  // U = V = I, so R = I and the batch contributes a translation-only step
  const float c = nrm == 0.0f ? 1.0f : fdiv(a, nrm), s = nrm == 0.0f ? 0.0f : fdiv(b, nrm);
  r[0][0] = c;
  r[0][1] = -s;
  r[0][2] = 0.0f;
  r[1][0] = s;
  r[1][1] = c;
  r[1][2] = 0.0f;
  r[2][0] = 0.0f;
  r[2][1] = 0.0f;
  r[2][2] = 1.0f;
}

// 3-D Procrustes: the proper rotation maximising trace(R H) = V diag(1, 1, det) U^T of H = U S V^T
// (icp.h:160-177), V from the eigen-decomposition of H^T H by cyclic Jacobi rotations in double
VBX_HD void icp_rotation_from_h3(const float hf[3][3], float r[3][3]) {
  double a[3][3], b[3][3], v[3][3];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) a[i][j] = hf[i][j];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      double s = 0;
      for (int k = 0; k < 3; ++k) s += a[k][i] * a[k][j];
      b[i][j] = s;
      v[i][j] = i == j ? 1.0 : 0.0;
    }
  for (int sweep = 0; sweep < 60; ++sweep) {
    double off = 0, diag = 0;
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) {
        if (i == j) {
          diag += b[i][j] * b[i][j];
        } else {
          off += b[i][j] * b[i][j];
        }
      }
    if (!(off > 1e-60) || off <= 1e-32 * diag) break;
    for (int p = 0; p < 2; ++p)
      for (int q = p + 1; q < 3; ++q) {
        if (b[p][q] == 0.0) continue;
        const double theta = (b[q][q] - b[p][p]) / (2.0 * b[p][q]);
        const double t = (theta >= 0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
        const double c = 1.0 / sqrt(t * t + 1.0), sn = t * c;
        for (int k = 0; k < 3; ++k) {
          const double bkp = b[k][p], bkq = b[k][q];
          b[k][p] = c * bkp - sn * bkq;
          b[k][q] = sn * bkp + c * bkq;
        }
        for (int k = 0; k < 3; ++k) {
          const double bpk = b[p][k], bqk = b[q][k];
          b[p][k] = c * bpk - sn * bqk;
          b[q][k] = sn * bpk + c * bqk;
        }
        for (int k = 0; k < 3; ++k) {
          const double vkp = v[k][p], vkq = v[k][q];
          v[k][p] = c * vkp - sn * vkq;
          v[k][q] = sn * vkp + c * vkq;
        }
      }
  }
  int order[3] = {0, 1, 2};
  for (int i = 0; i < 3; ++i)
    for (int j = i + 1; j < 3; ++j)
      if (b[order[j]][order[j]] > b[order[i]][order[i]]) {
        const int tmp = order[i];
        order[i] = order[j];
        order[j] = tmp;
      }
  double u[3][3], vs[3][3], sv[3];
  for (int c = 0; c < 3; ++c) {
    const double l = b[order[c]][order[c]];
    sv[c] = sqrt(l > 0 ? l : 0.0);
    for (int k = 0; k < 3; ++k) vs[k][c] = v[k][order[c]];
  }
  // The eigenvalues of H^T H carry an absolute error of about 1e-16 s1^2, so a singular value s_c taken
  // from them is off by a relative 1e-16 (s1 / s_c)^2, and H v_c / s_c is a unit vector orthogonal to the
  // other columns to float accuracy (6e-8) only while s_c > ~4e-5 s1; at 1e-4 s1 the error is 1e-8.  Planar
  // matched points (rank-2 H) leave s3 ~ 1e-8 s1 of rounding noise, collinear ones s2 too: columns below
  // 1e-4 s1 are completed instead of divided by their s.
  int good = 0;
  for (int c = 0; c < 3; ++c) {
    if (sv[c] > 1e-4 * sv[0] && sv[c] > 0) {
      for (int i = 0; i < 3; ++i) {
        double s = 0;
        for (int k = 0; k < 3; ++k) s += a[i][k] * vs[k][c];
        u[i][c] = s / sv[c];
      }
      good = c + 1;
    } else {
      break;
    }
  }
  // Completion of column c: H v_c made orthogonal to the columns before it and normalised (its direction
  // and sign are right wherever s_c is above the rounding noise of H v_c, ~1e-16 s1), else (rank < 2, or
  // H = 0) the first unit vector e_k that is not in the span of those columns, made orthogonal to them.
  for (int c = good; c < 3; ++c)
    for (int e = -1; e < 3; ++e) {
      double w[3];
      for (int i = 0; i < 3; ++i) w[i] = e < 0 ? a[i][0] * vs[0][c] + a[i][1] * vs[1][c] + a[i][2] * vs[2][c] : (i == e ? 1.0 : 0.0);
      for (int p = 0; p < c; ++p) {
        double dp = 0;
        for (int i = 0; i < 3; ++i) dp += w[i] * u[i][p];
        for (int i = 0; i < 3; ++i) w[i] -= dp * u[i][p];
      }
      const double nn = w[0] * w[0] + w[1] * w[1] + w[2] * w[2];
      if (nn > (e < 0 ? 1e-24 * sv[0] * sv[0] : 0.1)) {
        for (int i = 0; i < 3; ++i) u[i][c] = w[i] / sqrt(nn);
        break;
      }
    }
  float uf[3][3], vf[3][3];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      uf[i][j] = (float)u[i][j];
      vf[i][j] = (float)vs[i][j];
    }
  const float du = uf[0][0] * (uf[1][1] * uf[2][2] - uf[1][2] * uf[2][1]) - uf[0][1] * (uf[1][0] * uf[2][2] - uf[1][2] * uf[2][0]) +
                   uf[0][2] * (uf[1][0] * uf[2][1] - uf[1][1] * uf[2][0]);
  const float dv = vf[0][0] * (vf[1][1] * vf[2][2] - vf[1][2] * vf[2][1]) - vf[0][1] * (vf[1][0] * vf[2][2] - vf[1][2] * vf[2][0]) +
                   vf[0][2] * (vf[1][0] * vf[2][1] - vf[1][1] * vf[2][0]);
  if (du * dv < 0.0f)
    for (int i = 0; i < 3; ++i) vf[i][2] = vf[i][2] * -1.0f;
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) r[i][j] = vf[i][0] * uf[j][0] + vf[i][1] * uf[j][1] + vf[i][2] * uf[j][2];
}

// minkindr's Rotation::isValidRotationMatrix: |det R - 1| and every |(R R^T - I)_ij| within 1000 float
// epsilons (det by cofactors along the first row, R R^T by rows, summed in order; its coefficients (i, j)
// and (j, i) are the same products in the same order, so the upper triangle decides)
VBX_HD bool icp_is_valid_rotation(const float m[3][3]) {
  const float thr = 1000.0f * FLT_EPSILON;
  const float det = m[0][0] * (m[1][1] * m[2][2] - m[1][2] * m[2][1]) - m[0][1] * (m[1][0] * m[2][2] - m[1][2] * m[2][0]) +
                    m[0][2] * (m[1][0] * m[2][1] - m[1][1] * m[2][0]);
  if (fabsf(det - 1.0f) > thr) return false;
  for (int i = 0; i < 3; ++i)
    for (int j = i; j < 3; ++j) {
      const float e = m[i][0] * m[j][0] + m[i][1] * m[j][1] + m[i][2] * m[j][2] - (i == j ? 1.0f : 0.0f);
      if (fabsf(e) > thr) return false;
    }
  return true;
}

// getRotationFromMatchedPoints: the batch's rotation and whether ICP fuses it, i.e. R is finite and a
// valid rotation matrix (icp.h:183-189)
VBX_HD bool icp_rotation(const float h[3][3], bool refine_roll_pitch, float r[3][3]) {
  if (!refine_roll_pitch) {
    icp_rotation_2d(h, r);
  } else {
    icp_rotation_from_h3(h, r);
  }
  float sum = 0.0f;
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) sum += r[i][j];
  return isfinite(sum) && icp_is_valid_rotation(r);
}

// runThread's fusion of one batch's step `delta`, weighted by its information `info`, into the running pose
// `cur`; `base` accumulates the information fused so far (icp.cc:195-213)
VBX_HD void icp_fuse(IcpSE3& cur, float base[6], const IcpSE3& delta, const float info[6], float eps4_f, double eps4_d) {
  const IcpSE3 t_temp = icp_mul(delta, cur);
  IcpSE3 d = icp_mul(icp_inv(cur), t_temp);
  const F3 w3 = icp_quat_log(d.q, eps4_f);
  const float lg[6] = {d.t.x, d.t.y, d.t.z, w3.x, w3.y, w3.z};
  float wl[6];
  for (int i = 0; i < 6; ++i) {
    const float weight = fdiv(info[i], fadd(base[i], info[i]));
    wl[i] = fmul(weight, lg[i]);
    base[i] = fadd(base[i], info[i]);
  }
  d.q = icp_quat_exp(f3(wl[3], wl[4], wl[5]), eps4_d);
  d.t = f3(wl[0], wl[1], wl[2]);
  cur = icp_mul(cur, d);
}

}  // namespace vbx
