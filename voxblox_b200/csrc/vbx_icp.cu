// ICP pose refinement against the device-resident TSDF map (SURVEY.md section 8f N4).
//
// Reference: voxblox::ICP (include/voxblox/alignment/icp.h:72-233, src/alignment/icp.cc:43-261) with
// Interpolator<TsdfVoxel>'s nearest-voxel paths (interpolator/interpolator_inl.h:14-22, 48-77, 330-345;
// icp.cc:126-128 selects them).  The algorithm is a CHAIN: the point order is shuffled, mini batches of
// `mini_batch_size` points are matched against the TSDF one after the other, and every batch's
// least-squares transform is fused into the running pose, weighted by an information estimate, before
// the next batch of the same thread is matched (icp.cc:171-217).  With N/2/20 ~ 6500 links for a
// 640 x 480 cloud the work per link is tiny (20 points x 7 voxel reads, a 2 x 2 or 3 x 3 Procrustes
// problem, an SE(3) log / exp) and strictly ordered, so the device formulation is latency-minded:
//
//   * ONE thread block; warp w plays reference thread w (`num_threads` of them, <= 32) under the
//     round-robin schedule documented in include/voxblox_b200.h;
//   * matching: one lane per point of the batch -- pose transform, 7 independent block-hash probes +
//     voxel reads in flight per lane, central-difference gradient, target point -- into shared memory;
//   * reduction: the information vector, the two centroids and the cross-covariance are summed IN THE
//     REFERENCE'S ORDER (sequentially over the matched points), one lane per scalar, so the sums are
//     the reference's sums and only the library functions (asin / acos / sin / cos) can differ;
//   * fusion: thread 0 applies the fusions of the round in warp order.
//
// Arithmetic: float32 with one rounding per operation (the library is built with -fmad=false), in the
// operation order of the reference's Eigen / minkindr expressions.  The 2-D
// Procrustes rotation (refine_roll_pitch = false) uses the closed form atan2(h01 - h10, h00 + h11) of
// V diag(1, det) U^T; the 3-D one an SVD by Jacobi rotations on H^T H in double.
#include <algorithm>
#include <cmath>
#include <limits>
#include <numeric>
#include <random>
#include <vector>

#include "vbx_engine.h"
#include "vbx_hash.cuh"
#include "vbx_math.cuh"

namespace vbx {

struct IcpParams {
  float voxel_size, voxel_size_inv, block_size, block_size_inv;
  int vps, L;
  int refine_roll_pitch, mb, threads, min_matches;
  float keep_thr;  // subsample_keep_ratio * float(n)
  float tw, rw;
  float q[4], t[3];
  unsigned long long n;
  float eps4_f;   // epsilon^(1/4), float
  double eps4_d;  // epsilon^(1/4), double
};

struct IcpQuat {
  float w, x, y, z;
};
struct IcpSE3 {
  IcpQuat q;
  F3 t;
};

__device__ __forceinline__ IcpQuat icp_qmul(const IcpQuat& a, const IcpQuat& b) {
  IcpQuat r;
  r.w = a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z;
  r.x = a.w * b.x + a.x * b.w + a.y * b.z - a.z * b.y;
  r.y = a.w * b.y + a.y * b.w + a.z * b.x - a.x * b.z;
  r.z = a.w * b.z + a.z * b.w + a.x * b.y - a.y * b.x;
  return r;
}
__device__ __forceinline__ F3 icp_qrot(const IcpQuat& q, F3 p) {
  const F3 qv = f3(q.x, q.y, q.z);
  F3 uv = cross3(qv, p);
  uv = add3(uv, uv);
  return add3(add3(p, scale3(uv, q.w)), cross3(qv, uv));
}
__device__ __forceinline__ IcpSE3 icp_mul(const IcpSE3& a, const IcpSE3& b) {
  IcpSE3 r;
  r.q = icp_qmul(a.q, b.q);
  r.t = add3(a.t, icp_qrot(a.q, b.t));
  return r;
}
__device__ __forceinline__ IcpSE3 icp_inv(const IcpSE3& a) {
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
__device__ inline IcpQuat icp_quat_from_matrix(const float m[3][3]) {
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
// minkindr RotationQuaternion::log / exp
__device__ inline F3 icp_quat_log(const IcpQuat& q, float eps4_f) {
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
__device__ inline IcpQuat icp_quat_exp(F3 d, double eps4_d) {
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

// proper rotation maximising trace(R H) = V diag(1, 1, det) U^T of H = U S V^T (icp.h:160-177)
__device__ inline void icp_rotation_from_h3(const float hf[3][3], float r[3][3]) {
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
  int good = 0;
  for (int c = 0; c < 3; ++c) {
    if (sv[c] > 1e-12 * (sv[0] > 0 ? sv[0] : 1.0) && sv[c] > 0) {
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
  for (int c = good; c < 3; ++c)
    for (int e = 0; e < 3; ++e) {
      double w[3] = {e == 0 ? 1.0 : 0.0, e == 1 ? 1.0 : 0.0, e == 2 ? 1.0 : 0.0};
      for (int p = 0; p < c; ++p) {
        double dp = 0;
        for (int i = 0; i < 3; ++i) dp += w[i] * u[i][p];
        for (int i = 0; i < 3; ++i) w[i] -= dp * u[i][p];
      }
      const double nn = w[0] * w[0] + w[1] * w[1] + w[2] * w[2];
      if (nn > 0.1) {
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

// Interpolator::getNearestDistance (interpolator_inl.h:330-345) on the device map: the block by
// Layer::computeBlockIndexFromCoordinates (core/layer.h:128-131), the voxel by
// Block::computeTruncatedVoxelIndexFromCoordinates (core/block_inl.h:30-40).
// returns 0: no block, 1: block but voxel unobserved (weight <= 1e-6), 2: observed; *d = voxel distance
__device__ __forceinline__ int icp_nearest(const Tables& tab, const IcpParams& P, F3 p, float* d) {
  const I3 bi = grid_index(p, P.block_size_inv);
  const uint32_t hp = find_block(tab, pack3(bi.x, bi.y, bi.z));
  if (hp == 0xffffffffu) return 0;
  const int32_t slot = tab.hslot[hp];
  if (slot < 0) return 0;
  const F3 origin = f3(fmul((float)bi.x, P.block_size), fmul((float)bi.y, P.block_size), fmul((float)bi.z, P.block_size));
  const I3 vi = grid_index(sub3(p, origin), P.voxel_size_inv);
  const int mx = P.vps - 1;
  const int x = max(min(vi.x, mx), 0), y = max(min(vi.y, mx), 0), z = max(min(vi.z, mx), 0);
  const TsdfVoxel* v = tab.tsdf + (((size_t)slot << (3 * P.L)) + (size_t)(x + P.vps * (y + P.vps * z)));
  *d = v->distance;
  return (double)v->weight > 1e-6 ? 2 : 1;
}

constexpr int kIcpRec = 13;  // floats per matched point in shared memory: flag, p (3), target (3), info terms (6)

__global__ void __launch_bounds__(1024) k_icp(Tables tab, IcpParams P, const float* __restrict__ xyz,
                                              const uint32_t* __restrict__ perm, float* __restrict__ out) {
  extern __shared__ float smem[];
  const int T = P.threads, mb = P.mb;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* rec = smem + (size_t)warp * mb * kIcpRec;         // this warp's batch
  float* snap = smem + (size_t)T * mb * kIcpRec;           // [T][7] pose snapshots
  float* res = snap + T * 7;                               // [T][14] step results: ok, q (4), t (3), info (6)
  __shared__ float s_cur[7], s_base[6];
  __shared__ unsigned long long s_updates;
  if (threadIdx.x == 0) {
    for (int i = 0; i < 4; ++i) s_cur[i] = P.q[i];
    for (int i = 0; i < 3; ++i) s_cur[4 + i] = P.t[i];
    for (int i = 0; i < 3; ++i) {
      s_base[i] = P.tw;
      s_base[3 + i] = P.rw;
    }
    s_updates = 0;
  }
  if (lane < 7) snap[warp * 7 + lane] = lane < 4 ? P.q[lane] : P.t[lane - 4];
  __syncthreads();

  for (unsigned long long round = 0;; ++round) {
    // atomic_idx_.fetch_add in thread order (icp.cc:185-188): starts grow with the warp index, so the
    // round is empty exactly when warp 0 draws past the limit
    const unsigned long long start0 = round * (unsigned long long)T * (unsigned long long)mb;
    if ((float)start0 > P.keep_thr) break;
    const unsigned long long start = start0 + (unsigned long long)warp * (unsigned long long)mb;
    const bool has_job = !((float)start > P.keep_thr);
    if (has_job) {
      IcpSE3 Tw;
      Tw.q.w = snap[warp * 7 + 0];
      Tw.q.x = snap[warp * 7 + 1];
      Tw.q.y = snap[warp * 7 + 2];
      Tw.q.z = snap[warp * 7 + 3];
      Tw.t = f3(snap[warp * 7 + 4], snap[warp * 7 + 5], snap[warp * 7 + 6]);
      const unsigned long long end = min(P.n, start + (unsigned long long)mb);  // icp.cc:122-123
      const int cnt = end > start ? (int)(end - start) : 0;
      // ---- matchPoints (icp.cc:104-151), one lane per point
      for (int i = lane; i < cnt; i += 32) {
        const uint32_t src_i = perm[start + i];
        const F3 ps = f3(xyz[3 * (size_t)src_i], xyz[3 * (size_t)src_i + 1], xyz[3 * (size_t)src_i + 2]);
        const F3 p = add3(icp_qrot(Tw.q, ps), Tw.t);
        float d0, dm[3], dp[3];
        const int s0 = icp_nearest(tab, P, p, &d0);
        int ok = s0 == 2;
        // getGradient (interpolator_inl.h:48-77): every neighbour must be observed
#pragma unroll
        for (int a = 0; a < 3; ++a) {
          F3 qm = p, qp = p;
          const float off = P.voxel_size;
          if (a == 0) {
            qm.x = fadd(p.x, -off);
            qp.x = fadd(p.x, off);
          } else if (a == 1) {
            qm.y = fadd(p.y, -off);
            qp.y = fadd(p.y, off);
          } else {
            qm.z = fadd(p.z, -off);
            qp.z = fadd(p.z, off);
          }
          ok &= icp_nearest(tab, P, qm, &dm[a]) == 2;
          ok &= icp_nearest(tab, P, qp, &dp[a]) == 2;
        }
        float* r = rec + i * kIcpRec;
        float flag = 0.0f;
        if (ok) {
          const float den = fmul(2.0f, P.voxel_size);
          // grad(i) = (0 + d(-) * -1) + d(+) * 1, then / (2 voxel_size)
          F3 g = f3(fdiv(fadd(fadd(0.0f, fmul(dm[0], -1.0f)), fmul(dp[0], 1.0f)), den),
                    fdiv(fadd(fadd(0.0f, fmul(dm[1], -1.0f)), fmul(dp[1], 1.0f)), den),
                    fdiv(fadd(fadd(0.0f, fmul(dm[2], -1.0f)), fmul(dp[2], 1.0f)), den));
          if (dot3(g, g) > 0.1f) {  // kMinGradMag, icp.cc:114,130
            g = unit3(g);
            const F3 q = sub3(p, Tw.t);  // addNormalizedPointInfo(point_tsdf - T.getPosition(), gradient) (icp.cc:82-102)
            r[7] = 2.0f * (g.x * g.x);
            r[8] = 2.0f * (g.y * g.y);
            r[9] = 2.0f * (g.z * g.z);
            r[10] = 2.0f * (q.y * q.y * g.z * g.z + q.z * q.z * g.y * g.y);
            r[11] = 2.0f * (q.x * q.x * g.z * g.z + q.z * q.z * g.x * g.x);
            r[12] = 2.0f * (q.x * q.x * g.y * g.y + q.y * q.y * g.x * g.x);
            const I3 vidx = grid_index(p, P.voxel_size_inv);
            const F3 centre = f3(center_coord(vidx.x, P.voxel_size), center_coord(vidx.y, P.voxel_size),
                                 center_coord(vidx.z, P.voxel_size));
            const float dist = fadd(d0, dot3(g, sub3(p, centre)));
            const F3 tg = sub3(p, scale3(g, dist));
            r[1] = p.x;
            r[2] = p.y;
            r[3] = p.z;
            r[4] = tg.x;
            r[5] = tg.y;
            r[6] = tg.z;
            flag = 1.0f;
          }
        }
        r[0] = flag;
      }
      __syncwarp();
      // ---- sums in the reference's order: lanes 0-5 information, 6-8 source sum, 9-11 target sum
      float acc = lane < 6 ? VBX_EPS : 0.0f;
      int nv = 0;
      if (lane < 12) {
        const int col = lane < 6 ? 7 + lane : lane - 5;  // 7..12 | 1..3 | 4..6
        for (int i = 0; i < cnt; ++i) {
          const float* r = rec + i * kIcpRec;
          if (r[0] != 0.0f) {
            acc = (lane >= 6 && nv == 0) ? r[col] : fadd(acc, r[col]);
            ++nv;
          }
        }
      }
      nv = __shfl_sync(0xffffffffu, nv, 0);
      const bool enough = nv >= P.min_matches;  // icp.cc:161-164
      // centroids (icp.cc:58-63)
      const float mean = lane >= 6 && lane < 12 ? fdiv(acc, (float)nv) : 0.0f;
      const float sc[3] = {__shfl_sync(0xffffffffu, mean, 6), __shfl_sync(0xffffffffu, mean, 7), __shfl_sync(0xffffffffu, mean, 8)};
      const float tc[3] = {__shfl_sync(0xffffffffu, mean, 9), __shfl_sync(0xffffffffu, mean, 10), __shfl_sync(0xffffffffu, mean, 11)};
      float info[6];
#pragma unroll
      for (int k = 0; k < 6; ++k) info[k] = __shfl_sync(0xffffffffu, acc, k);
      // H = src_demean * tgt_demean^T (icp.h:156-157), lane = 3 i + j
      float hacc = 0.0f;
      if (enough && lane < 9) {
        const int hi = lane / 3, hj = lane % 3;
        for (int i = 0; i < cnt; ++i) {
          const float* r = rec + i * kIcpRec;
          if (r[0] != 0.0f) hacc = fadd(hacc, fmul(fsub(r[1 + hi], sc[hi]), fsub(r[4 + hj], tc[hj])));
        }
      }
      float h[3][3];
#pragma unroll
      for (int k = 0; k < 9; ++k) h[k / 3][k % 3] = __shfl_sync(0xffffffffu, hacc, k);
      if (lane == 0) {
        float* o = res + warp * 14;
        float ok = 0.0f;
        if (enough) {
          float r[3][3] = {{1, 0, 0}, {0, 1, 0}, {0, 0, 1}};
          if (!P.refine_roll_pitch) {
            const float a = fadd(h[0][0], h[1][1]), b = fsub(h[0][1], h[1][0]);
            const float nrm = fsqrt(fadd(fmul(a, a), fmul(b, b)));
            const float c = fdiv(a, nrm), s = fdiv(b, nrm);
            r[0][0] = c;
            r[0][1] = -s;
            r[1][0] = s;
            r[1][1] = c;
          } else {
            icp_rotation_from_h3(h, r);
          }
          float sum = 0.0f;
          for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j) sum += r[i][j];
          if (isfinite(sum)) {  // icp.h:183-186
            const IcpQuat dq = icp_quat_from_matrix(r);
            const F3 dt = sub3(f3(tc[0], tc[1], tc[2]), icp_qrot(dq, f3(sc[0], sc[1], sc[2])));  // icp.cc:74-77
            o[1] = dq.w;
            o[2] = dq.x;
            o[3] = dq.y;
            o[4] = dq.z;
            o[5] = dt.x;
            o[6] = dt.y;
            o[7] = dt.z;
            for (int k = 0; k < 6; ++k) o[8 + k] = info[k];
            ok = 1.0f;
          }
        }
        o[0] = ok;
      }
    } else if (lane == 0) {
      res[warp * 14] = 0.0f;
    }
    __syncthreads();
    // ---- fusion in thread order (icp.cc:195-213)
    if (threadIdx.x == 0) {
      IcpSE3 cur;
      cur.q.w = s_cur[0];
      cur.q.x = s_cur[1];
      cur.q.y = s_cur[2];
      cur.q.z = s_cur[3];
      cur.t = f3(s_cur[4], s_cur[5], s_cur[6]);
      for (int w = 0; w < T; ++w) {
        const float* o = res + w * 14;
        if (o[0] == 0.0f) continue;
        IcpSE3 delta;
        delta.q.w = o[1];
        delta.q.x = o[2];
        delta.q.y = o[3];
        delta.q.z = o[4];
        delta.t = f3(o[5], o[6], o[7]);
        const IcpSE3 t_temp = icp_mul(delta, cur);
        IcpSE3 d = icp_mul(icp_inv(cur), t_temp);
        const F3 w3 = icp_quat_log(d.q, P.eps4_f);
        const float lg[6] = {d.t.x, d.t.y, d.t.z, w3.x, w3.y, w3.z};
        float wl[6];
        for (int i = 0; i < 6; ++i) {
          const float weight = fdiv(o[8 + i], fadd(s_base[i], o[8 + i]));
          wl[i] = fmul(weight, lg[i]);
          s_base[i] = fadd(s_base[i], o[8 + i]);
        }
        d.q = icp_quat_exp(f3(wl[3], wl[4], wl[5]), P.eps4_d);
        d.t = f3(wl[0], wl[1], wl[2]);
        cur = icp_mul(cur, d);
        float* sp = snap + w * 7;
        sp[0] = cur.q.w;
        sp[1] = cur.q.x;
        sp[2] = cur.q.y;
        sp[3] = cur.q.z;
        sp[4] = cur.t.x;
        sp[5] = cur.t.y;
        sp[6] = cur.t.z;
        ++s_updates;
      }
      s_cur[0] = cur.q.w;
      s_cur[1] = cur.q.x;
      s_cur[2] = cur.q.y;
      s_cur[3] = cur.q.z;
      s_cur[4] = cur.t.x;
      s_cur[5] = cur.t.y;
      s_cur[6] = cur.t.z;
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    for (int i = 0; i < 7; ++i) out[i] = s_cur[i];
    out[7] = 0.0f;
    *reinterpret_cast<unsigned long long*>(out + 8) = s_updates;
  }
}

void icp_destroy(vbx_ctx* c) {
  if (c->icp_perm_dev) cudaFree(c->icp_perm_dev);
  if (c->icp_perm_host) cudaFreeHost(c->icp_perm_host);
  if (c->icp_out_dev) cudaFree(c->icp_out_dev);
  if (c->icp_out_host) cudaFreeHost(c->icp_out_host);
  if (c->icp_points_dev) cudaFree(c->icp_points_dev);
  c->icp_perm_dev = nullptr;
  c->icp_perm_host = nullptr;
  c->icp_out_dev = nullptr;
  c->icp_out_host = nullptr;
  c->icp_points_dev = nullptr;
  c->icp_cap = 0;
}

int icp_run(vbx_ctx* c, const vbx_icp_config* cfg, const float* points, int on_device, uint64_t n, const float q[4],
            const float t[3], uint32_t seed, float out_q[4], float out_t[3], uint64_t* num_updates) {
  if (cfg->num_threads < 1 || cfg->num_threads > 32) return fail(c, VBX_E_INVALID, "icp: num_threads must be 1..32");
  if (cfg->mini_batch_size < 1) return fail(c, VBX_E_INVALID, "icp: mini_batch_size must be positive");
  if (n >= (1ull << 31)) return fail(c, VBX_E_CAPACITY, "icp: too many points");
  const size_t smem = ((size_t)cfg->num_threads * cfg->mini_batch_size * kIcpRec + (size_t)cfg->num_threads * 21) * sizeof(float);
  if (smem > 200 * 1024) return fail(c, VBX_E_CAPACITY, "icp: num_threads * mini_batch_size too large for shared memory");
  if (n > c->icp_cap || !c->icp_out_dev) {
    icp_destroy(c);
    const uint64_t cap = std::max<uint64_t>(n, 1024);
    VBX_CUDA(c, cudaMalloc(reinterpret_cast<void**>(&c->icp_perm_dev), cap * sizeof(uint32_t)));
    VBX_CUDA(c, cudaHostAlloc(reinterpret_cast<void**>(&c->icp_perm_host), cap * sizeof(uint32_t), cudaHostAllocDefault));
    VBX_CUDA(c, cudaMalloc(reinterpret_cast<void**>(&c->icp_points_dev), cap * 3 * sizeof(float)));
    VBX_CUDA(c, cudaMalloc(reinterpret_cast<void**>(&c->icp_out_dev), 16 * sizeof(float)));
    VBX_CUDA(c, cudaHostAlloc(reinterpret_cast<void**>(&c->icp_out_host), 16 * sizeof(float), cudaHostAllocDefault));
    c->icp_cap = cap;
  }
  cudaStream_t s = c->stream;
  const float* d_points = points;
  if (!on_device && n) {
    VBX_CUDA(c, cudaMemcpyAsync(c->icp_points_dev, points, n * 3 * sizeof(float), cudaMemcpyHostToDevice, s));
    d_points = c->icp_points_dev;
  }
  // the reference's shuffle (icp.cc:229-233) is a function of (n, seed) only: run the C++ library's own
  // std::shuffle on the index sequence while the cloud is on its way to the device
  std::iota(c->icp_perm_host, c->icp_perm_host + n, 0u);
  std::shuffle(c->icp_perm_host, c->icp_perm_host + n, std::default_random_engine(seed));
  if (n) VBX_CUDA(c, cudaMemcpyAsync(c->icp_perm_dev, c->icp_perm_host, n * sizeof(uint32_t), cudaMemcpyHostToDevice, s));

  IcpParams P;
  P.voxel_size = c->voxel_size;
  P.voxel_size_inv = c->voxel_size_inv;
  P.block_size = c->voxel_size * (float)(size_t)c->vps;             // Layer ctor, core/layer.h:39
  P.block_size_inv = (float)(1.0 / (double)P.block_size);           // core/layer.h:41
  P.vps = c->vps;
  P.L = c->L;
  P.refine_roll_pitch = cfg->refine_roll_pitch ? 1 : 0;
  P.mb = cfg->mini_batch_size;
  P.threads = cfg->num_threads;
  P.min_matches = std::max(3, (int)((float)cfg->mini_batch_size * cfg->min_match_ratio));  // icp.cc:161-162
  P.keep_thr = cfg->subsample_keep_ratio * (float)n;                                         // icp.cc:186
  P.tw = cfg->inital_translation_weighting;
  P.rw = cfg->inital_rotation_weighting;
  for (int i = 0; i < 4; ++i) P.q[i] = q[i];
  for (int i = 0; i < 3; ++i) P.t[i] = t[i];
  P.n = n;
  P.eps4_f = std::pow(std::numeric_limits<float>::epsilon(), 0.25f);
  P.eps4_d = std::pow(std::numeric_limits<double>::epsilon(), 0.25);
  if (smem > 48 * 1024) {
    VBX_CUDA(c, cudaFuncSetAttribute(k_icp, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  }
  k_icp<<<1, 32 * cfg->num_threads, smem, s>>>(c->tab, P, d_points, c->icp_perm_dev, c->icp_out_dev);
  ++c->launches;
  VBX_CUDA(c, cudaGetLastError());
  VBX_CUDA(c, cudaMemcpyAsync(c->icp_out_host, c->icp_out_dev, 16 * sizeof(float), cudaMemcpyDeviceToHost, s));
  VBX_CUDA(c, cudaStreamSynchronize(s));
  for (int i = 0; i < 4; ++i) out_q[i] = c->icp_out_host[i];
  for (int i = 0; i < 3; ++i) out_t[i] = c->icp_out_host[4 + i];
  if (num_updates) *num_updates = *reinterpret_cast<const unsigned long long*>(c->icp_out_host + 8);
  return VBX_OK;
}

}  // namespace vbx
