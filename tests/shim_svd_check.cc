// The test build's stand-in JacobiSVD (oracle/shim/Eigen/Core) on its own, with no reference source, for
// tests/test_icp_math_cpu.py: U and V of N x N matrices (N = 2, 3), row-major in and out.
// Build: g++ -std=c++14 -O2 -ffp-contract=off -fPIC -shared -I oracle/shim
#include <Eigen/Core>

#include <cstdint>

namespace {
template <int N>
void svd(uint32_t n, const float* h, float* u, float* v) {
  for (uint32_t i = 0; i < n; ++i) {
    Eigen::Matrix<float, N, N> m;
    for (int r = 0; r < N; ++r)
      for (int c = 0; c < N; ++c) m(r, c) = h[N * N * (size_t)i + N * r + c];
    const Eigen::JacobiSVD<Eigen::Matrix<float, N, N> > s(m, Eigen::ComputeFullU | Eigen::ComputeFullV);
    for (int r = 0; r < N; ++r)
      for (int c = 0; c < N; ++c) {
        u[N * N * (size_t)i + N * r + c] = s.matrixU()(r, c);
        v[N * N * (size_t)i + N * r + c] = s.matrixV()(r, c);
      }
  }
}
}  // namespace

extern "C" void shim_svd(int dim, uint32_t n, const float* h, float* u, float* v) {
  if (dim == 2) svd<2>(n, h, u, v);
  if (dim == 3) svd<3>(n, h, u, v);
}
