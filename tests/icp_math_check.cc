// Host build of ICP's per-batch arithmetic (voxblox_b200/csrc/vbx_icp_math.cuh) for
// tests/test_icp_math_cpu.py.  icp_math_batch does per item what k_icp_debug_solve (vbx_icp.cu) does per
// device thread, so tests/test_icp_math_gpu.py can compare the two bit for bit.
// Build: g++ -std=c++17 -O2 -ffp-contract=off -fPIC -shared (one IEEE rounding per operation).
#include <cmath>
#include <cstdint>
#include <limits>

#include "../voxblox_b200/csrc/vbx_icp_math.cuh"

using namespace vbx;

namespace {
const float kEps4F = std::pow(std::numeric_limits<float>::epsilon(), 0.25f);
const double kEps4D = std::pow(std::numeric_limits<double>::epsilon(), 0.25);
}  // namespace

extern "C" {

// h, m: 9 floats per item (row-major); q: 4 (w, x, y, z); w: 3.  Out: r (9), valid, q_out = quaternion of m (4),
// log_out = log(q) (3), exp_out = exp(w) (4)
void icp_math_batch(uint32_t n, int refine_roll_pitch, const float* h, const float* m, const float* q, const float* w,
                    float* r_out, int32_t* valid_out, float* q_out, float* log_out, float* exp_out) {
  for (uint32_t i = 0; i < n; ++i) {
    float hh[3][3], mm[3][3], r[3][3];
    for (int k = 0; k < 9; ++k) {
      hh[k / 3][k % 3] = h[9 * (size_t)i + k];
      mm[k / 3][k % 3] = m[9 * (size_t)i + k];
    }
    valid_out[i] = icp_rotation(hh, refine_roll_pitch != 0, r) ? 1 : 0;
    for (int k = 0; k < 9; ++k) r_out[9 * (size_t)i + k] = r[k / 3][k % 3];
    const IcpQuat qm = icp_quat_from_matrix(mm);
    const IcpQuat qi = {q[4 * (size_t)i], q[4 * (size_t)i + 1], q[4 * (size_t)i + 2], q[4 * (size_t)i + 3]};
    const F3 lg = icp_quat_log(qi, kEps4F);
    const IcpQuat ex = icp_quat_exp(f3(w[3 * (size_t)i], w[3 * (size_t)i + 1], w[3 * (size_t)i + 2]), kEps4D);
    const float qv[4] = {qm.w, qm.x, qm.y, qm.z}, lv[3] = {lg.x, lg.y, lg.z}, ev[4] = {ex.w, ex.x, ex.y, ex.z};
    for (int k = 0; k < 4; ++k) q_out[4 * (size_t)i + k] = qv[k];
    for (int k = 0; k < 3; ++k) log_out[3 * (size_t)i + k] = lv[k];
    for (int k = 0; k < 4; ++k) exp_out[4 * (size_t)i + k] = ev[k];
  }
}

// one fusion (icp_fuse) per item: cur = (q wxyz, t) 7 floats and base 6 floats updated in place; delta 7, info 6
void icp_fuse_batch(uint32_t n, float* cur, float* base, const float* delta, const float* info) {
  for (uint32_t i = 0; i < n; ++i) {
    float* c = cur + 7 * (size_t)i;
    const float* d = delta + 7 * (size_t)i;
    IcpSE3 T = {{c[0], c[1], c[2], c[3]}, f3(c[4], c[5], c[6])};
    const IcpSE3 D = {{d[0], d[1], d[2], d[3]}, f3(d[4], d[5], d[6])};
    icp_fuse(T, base + 6 * (size_t)i, D, info + 6 * (size_t)i, kEps4F, kEps4D);
    const float out[7] = {T.q.w, T.q.x, T.q.y, T.q.z, T.t.x, T.t.y, T.t.z};
    for (int k = 0; k < 7; ++k) c[k] = out[k];
  }
}

}  // extern "C"
