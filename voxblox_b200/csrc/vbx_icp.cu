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
// V diag(1, det) U^T; the 3-D one an SVD by Jacobi rotations on H^T H in double (vbx_icp_math.cuh).
#include <algorithm>
#include <cmath>
#include <limits>
#include <numeric>
#include <random>
#include <vector>

#include "vbx_engine.h"
#include "vbx_hash.cuh"
#include "vbx_icp_math.cuh"
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
          float r[3][3];
          if (icp_rotation(h, P.refine_roll_pitch != 0, r)) {
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
        icp_fuse(cur, s_base, delta, o + 8, P.eps4_f, P.eps4_d);
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

// vbx_debug_icp_solve: one thread per item runs the per-batch arithmetic of k_icp on caller-given inputs
__global__ void k_icp_debug_solve(uint32_t n, int refine_roll_pitch, float eps4_f, double eps4_d, const float* __restrict__ h,
                                  const float* __restrict__ m, const float* __restrict__ q, const float* __restrict__ w,
                                  float* __restrict__ r_out, int32_t* __restrict__ valid_out, float* __restrict__ q_out,
                                  float* __restrict__ log_out, float* __restrict__ exp_out) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float hh[3][3], mm[3][3], r[3][3];
  for (int k = 0; k < 9; ++k) {
    hh[k / 3][k % 3] = h[9 * (size_t)i + k];
    mm[k / 3][k % 3] = m[9 * (size_t)i + k];
  }
  valid_out[i] = icp_rotation(hh, refine_roll_pitch != 0, r) ? 1 : 0;
  for (int k = 0; k < 9; ++k) r_out[9 * (size_t)i + k] = r[k / 3][k % 3];
  const IcpQuat qm = icp_quat_from_matrix(mm);
  IcpQuat qi;
  qi.w = q[4 * (size_t)i];
  qi.x = q[4 * (size_t)i + 1];
  qi.y = q[4 * (size_t)i + 2];
  qi.z = q[4 * (size_t)i + 3];
  const F3 lg = icp_quat_log(qi, eps4_f);
  const IcpQuat ex = icp_quat_exp(f3(w[3 * (size_t)i], w[3 * (size_t)i + 1], w[3 * (size_t)i + 2]), eps4_d);
  const float qv[4] = {qm.w, qm.x, qm.y, qm.z}, lv[3] = {lg.x, lg.y, lg.z}, ev[4] = {ex.w, ex.x, ex.y, ex.z};
  for (int k = 0; k < 4; ++k) q_out[4 * (size_t)i + k] = qv[k];
  for (int k = 0; k < 3; ++k) log_out[3 * (size_t)i + k] = lv[k];
  for (int k = 0; k < 4; ++k) exp_out[4 * (size_t)i + k] = ev[k];
}

int icp_debug_solve(vbx_ctx* c, uint32_t n, int refine_roll_pitch, const float* h, const float* m, const float* q,
                    const float* w, float* r_out, int32_t* valid_out, float* q_out, float* log_out, float* exp_out) {
  if (!n) return VBX_OK;
  // one device allocation: h (9), m (9), q (4), w (3) in; r (9), q (4), log (3), exp (4) and valid out, per item
  const size_t nn = n;
  float* d = nullptr;
  Holdings scratch;
  VBX_CUDA(c, scratch.dev(&d, 46 * nn));
  float *dh = d, *dm = dh + 9 * nn, *dq = dm + 9 * nn, *dw = dq + 4 * nn;
  float *dr = dw + 3 * nn, *dqo = dr + 9 * nn, *dl = dqo + 4 * nn, *de = dl + 3 * nn;
  int32_t* dv = reinterpret_cast<int32_t*>(de + 4 * nn);
  cudaStream_t s = c->stream;
  const float* hin[4] = {h, m, q, w};
  float* din[4] = {dh, dm, dq, dw};
  const size_t width_in[4] = {9, 9, 4, 3};
  for (int k = 0; k < 4; ++k) {
    VBX_CUDA(c, cudaMemcpyAsync(din[k], hin[k], width_in[k] * nn * sizeof(float), cudaMemcpyHostToDevice, s));
  }
  k_icp_debug_solve<<<(n + 127) / 128, 128, 0, s>>>(n, refine_roll_pitch, std::pow(std::numeric_limits<float>::epsilon(), 0.25f),
                                                    std::pow(std::numeric_limits<double>::epsilon(), 0.25), dh, dm, dq, dw, dr, dv,
                                                    dqo, dl, de);
  ++c->launches;
  VBX_CUDA(c, cudaGetLastError());
  float* hout[4] = {r_out, q_out, log_out, exp_out};
  const float* dout[4] = {dr, dqo, dl, de};
  const size_t width_out[4] = {9, 4, 3, 4};
  for (int k = 0; k < 4; ++k) {
    VBX_CUDA(c, cudaMemcpyAsync(hout[k], dout[k], width_out[k] * nn * sizeof(float), cudaMemcpyDeviceToHost, s));
  }
  VBX_CUDA(c, cudaMemcpyAsync(valid_out, dv, nn * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
  VBX_CUDA(c, cudaStreamSynchronize(s));
  return VBX_OK;
}

int icp_run(vbx_ctx* c, const vbx_icp_config* cfg, const float* points, int on_device, uint64_t n, const float q[4],
            const float t[3], uint32_t seed, float out_q[4], float out_t[3], uint64_t* num_updates) {
  if (cfg->num_threads < 1 || cfg->num_threads > 32) return fail(c, VBX_E_INVALID, "icp: num_threads must be 1..32");
  if (cfg->mini_batch_size < 1) return fail(c, VBX_E_INVALID, "icp: mini_batch_size must be positive");
  if (n >= (1ull << 31)) return fail(c, VBX_E_CAPACITY, "icp: too many points");
  const size_t smem = ((size_t)cfg->num_threads * cfg->mini_batch_size * kIcpRec + (size_t)cfg->num_threads * 21) * sizeof(float);
  if (smem > 200 * 1024) return fail(c, VBX_E_CAPACITY, "icp: num_threads * mini_batch_size too large for shared memory");
  if (n > c->icp.cap || !c->icp.out_dev) {
    Holdings& h = c->icp.own;
    h.release();
    c->icp.cap = 0;
    const uint64_t cap = std::max<uint64_t>(n, 1024);
    VBX_CUDA(c, h.dev(&c->icp.perm_dev, cap));
    VBX_CUDA(c, h.host(&c->icp.perm_host, cap));
    VBX_CUDA(c, h.dev(&c->icp.points_dev, cap * 3));
    VBX_CUDA(c, h.dev(&c->icp.out_dev, 16));
    VBX_CUDA(c, h.host(&c->icp.out_host, 16));
    c->icp.cap = cap;
  }
  cudaStream_t s = c->stream;
  const float* d_points = points;
  if (!on_device && n) {
    VBX_CUDA(c, cudaMemcpyAsync(c->icp.points_dev, points, n * 3 * sizeof(float), cudaMemcpyHostToDevice, s));
    d_points = c->icp.points_dev;
  }
  // the reference's shuffle (icp.cc:229-233) is a function of (n, seed) only: run the C++ library's own
  // std::shuffle on the index sequence while the cloud is on its way to the device
  std::iota(c->icp.perm_host, c->icp.perm_host + n, 0u);
  std::shuffle(c->icp.perm_host, c->icp.perm_host + n, std::default_random_engine(seed));
  if (n) VBX_CUDA(c, cudaMemcpyAsync(c->icp.perm_dev, c->icp.perm_host, n * sizeof(uint32_t), cudaMemcpyHostToDevice, s));

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
  k_icp<<<1, 32 * cfg->num_threads, smem, s>>>(c->tab, P, d_points, c->icp.perm_dev, c->icp.out_dev);
  ++c->launches;
  VBX_CUDA(c, cudaGetLastError());
  VBX_CUDA(c, cudaMemcpyAsync(c->icp.out_host, c->icp.out_dev, 16 * sizeof(float), cudaMemcpyDeviceToHost, s));
  VBX_CUDA(c, cudaStreamSynchronize(s));
  for (int i = 0; i < 4; ++i) out_q[i] = c->icp.out_host[i];
  for (int i = 0; i < 3; ++i) out_t[i] = c->icp.out_host[4 + i];
  if (num_updates) *num_updates = *reinterpret_cast<const unsigned long long*>(c->icp.out_host + 8);
  return VBX_OK;
}

}  // namespace vbx
