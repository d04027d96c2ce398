// TEST INFRASTRUCTURE ONLY (oracle/): a single-threaded CPU restatement of the
// voxblox TSDF / ESDF integration hot path, written from the reference's
// behaviour (every function cites the reference file:line it follows; all paths
// are under /root/reference/voxblox).  It exists to CHECK the CUDA engine; it is
// never linked into, imported by or executed from the product (voxblox_b200/).
//
// Pinning: tests/test_oracle_pin.py runs this restatement and the reference's own
// sources (oracle/_ref/libvbx_ref.so = the verbatim .cc files compiled against
// oracle/shim/) on the same seeded scans and requires bit-identical layers, and
// replays the known-answer indexing vectors of test/test_tsdf_map.cc.  Committed
// digests under tests/golden/ pin it where /root/reference is absent.
//
// Arithmetic conventions restated from the reference's third-party deps (Eigen 3.3
// and ethz-asl/minkindr, both unpinned in voxblox_https.rosinstall:5-22):
//   sum of 3 coefficients  = c0 + (c1 + c2)            (Eigen Redux.h unroller)
//   normalized(v)          = v / sqrt(|v|^2), v if |v|^2 == 0   (Eigen Dot.h, 3.3)
//   q * v                  = v + w*(2 q.vec x v) + q.vec x (2 q.vec x v)
//   T * p                  = q * p + t                 (minkindr transform())
// Build: g++ -O2 -ffp-contract=off, no -march=native => one IEEE rounding per op.
#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <limits>
#include <memory>
#include <numeric>
#include <queue>
#include <random>
#include <unordered_map>
#include <unordered_set>
#include <utility>
#include <vector>

#include "vbo_api.h"
#include "../voxblox_b200/csrc/vbx_mc_tables.h"  // generated case table, pinned to the reference table by tests/test_mesh_cpu.py

namespace {

// ----------------------------------------------------------------------- 3-vectors
struct V3 {
  float x, y, z;
};
inline V3 operator+(V3 a, V3 b) { return {a.x + b.x, a.y + b.y, a.z + b.z}; }
inline V3 operator-(V3 a, V3 b) { return {a.x - b.x, a.y - b.y, a.z - b.z}; }
inline V3 operator*(V3 a, float s) { return {a.x * s, a.y * s, a.z * s}; }
inline V3 operator/(V3 a, float s) { return {a.x / s, a.y / s, a.z / s}; }
inline float dot3(V3 a, V3 b) { return a.x * b.x + (a.y * b.y + a.z * b.z); }
inline float sqnorm3(V3 a) { return dot3(a, a); }
inline float norm3(V3 a) { return std::sqrt(sqnorm3(a)); }
inline V3 unit3(V3 a) {
  const float z = sqnorm3(a);
  return z > 0.0f ? a / std::sqrt(z) : a;
}
inline V3 cross3(V3 a, V3 b) {
  return {a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x};
}

struct Pose {  // T_G_C
  float w, x, y, z;
  V3 t;
  V3 apply(V3 p) const {
    const V3 qv{x, y, z};
    V3 uv = cross3(qv, p);
    uv = uv + uv;
    return ((p + uv * w) + cross3(qv, uv)) + t;
  }
};

// --------------------------------------------------------------------- index types
struct I3 {  // AnyIndex / BlockIndex / VoxelIndex (core/common.h:48-51)
  int x, y, z;
  bool operator==(const I3& o) const { return x == o.x && y == o.y && z == o.z; }
};
struct L3 {  // LongIndex / GlobalIndex (core/common.h:53-54)
  int64_t x, y, z;
  bool operator==(const L3& o) const { return x == o.x && y == o.y && z == o.z; }
  bool operator!=(const L3& o) const { return !(*this == o); }
};
// core/block_hash.h:20-33 and :52-64: x + 17191 y + 17191^2 z, truncated to 32 bits.
struct HashI3 {
  size_t operator()(const I3& i) const {
    return static_cast<unsigned int>(static_cast<size_t>(i.x) + static_cast<size_t>(i.y) * 17191u +
                                     static_cast<size_t>(i.z) * (17191ull * 17191ull));
  }
};
struct HashL3 {
  size_t operator()(const L3& i) const {
    return static_cast<unsigned int>(static_cast<size_t>(i.x) + static_cast<size_t>(i.y) * 17191u +
                                     static_cast<size_t>(i.z) * (17191ull * 17191ull));
  }
};

constexpr float kEps = 1e-6f;  // kEpsilon / kFloatEpsilon, core/common.h:139-140

// core/common.h:153-159 (with a grid_size_inv) and :166-171 (pre-scaled point)
inline L3 gridIndex(V3 p, float inv) {
  return {static_cast<int64_t>(std::floor(p.x * inv + kEps)),
          static_cast<int64_t>(std::floor(p.y * inv + kEps)),
          static_cast<int64_t>(std::floor(p.z * inv + kEps))};
}
inline L3 gridIndexScaled(V3 p) {
  return {static_cast<int64_t>(std::floor(p.x + kEps)), static_cast<int64_t>(std::floor(p.y + kEps)),
          static_cast<int64_t>(std::floor(p.z + kEps))};
}
// core/common.h:186-193: (float(idx) + 0.5 [double]) * grid_size, rounded to float
inline V3 centerPoint(const L3& i, float grid) {
  return {static_cast<float>((static_cast<float>(i.x) + 0.5) * grid),
          static_cast<float>((static_cast<float>(i.y) + 0.5) * grid),
          static_cast<float>((static_cast<float>(i.z) + 0.5) * grid)};
}
// core/common.h:215-224
inline I3 blockOf(const L3& g, float vps_inv) {
  return {static_cast<int>(std::floor(static_cast<float>(g.x) * vps_inv)),
          static_cast<int>(std::floor(static_cast<float>(g.y) * vps_inv)),
          static_cast<int>(std::floor(static_cast<float>(g.z) * vps_inv))};
}
// core/common.h:233-243 and core/block_inl.h:12-27
inline size_t localLinear(const L3& g, int vps) {
  constexpr int64_t off = int64_t(1) << 31;  // "1 << (8*sizeof(int) - 1)" wraps to INT_MIN; & mask is the same
  const int lx = static_cast<int>((g.x + off) & (vps - 1));
  const int ly = static_cast<int>((g.y + off) & (vps - 1));
  const int lz = static_cast<int>((g.z + off) & (vps - 1));
  return static_cast<size_t>(lx + vps * (ly + lz * vps));
}
inline int signumf(float v) { return (v == 0) ? 0 : (v < 0 ? -1 : 1); }  // core/common.h:258

// -------------------------------------------------------------------------- voxels
struct Rgba {
  uint8_t r, g, b, a;
};
struct TsdfVox {  // core/voxel.h:12-16
  float distance = 0.0f;
  float weight = 0.0f;
  Rgba color{0, 0, 0, 0};
};
struct EsdfVox {  // core/voxel.h:18-37
  float distance = 0.0f;
  uint8_t observed = 0, hallucinated = 0, in_queue = 0, fixed = 0;
  int32_t parent[3] = {0, 0, 0};
};
static_assert(sizeof(TsdfVox) == 12 && sizeof(EsdfVox) == 20, "voxel layouts");

// core/common.h:105-125
inline Rgba blend(Rgba c1, float w1, Rgba c2, float w2) {
  const float total = w1 + w2;
  w1 /= total;
  w2 /= total;
  Rgba o;
  o.r = static_cast<uint8_t>(std::round(c1.r * w1 + c2.r * w2));
  o.g = static_cast<uint8_t>(std::round(c1.g * w1 + c2.g * w2));
  o.b = static_cast<uint8_t>(std::round(c1.b * w1 + c2.b * w2));
  o.a = static_cast<uint8_t>(std::round(c1.a * w1 + c2.a * w2));
  return o;
}

template <typename V>
struct Blk {
  std::vector<V> vox;
  uint8_t updated = 0;  // bit0 kMap, bit1 kMesh, bit2 kEsdf (core/block.h:15-18)
  explicit Blk(int vps) : vox(static_cast<size_t>(vps) * vps * vps) {}
};
template <typename V>
using BlockMap = std::unordered_map<I3, std::shared_ptr<Blk<V>>, HashI3>;

// ----------------------------------------------------------------------- ray caster
// integrator/integrator_utils.cc:72-179 (Amanatides-Woo in voxel units)
struct Dda {
  L3 cur{0, 0, 0};
  int sgn[3] = {0, 0, 0};
  float tnext[3] = {0, 0, 0}, tstep[3] = {0, 0, 0};
  unsigned int len = 0, step = 0;
  bool dead = false;

  Dda(V3 origin, V3 point_G, bool clearing, bool carving, float max_ray, float inv, float trunc,
      bool from_origin) {
    const V3 u = unit3(point_G - origin);
    V3 a, b;
    if (clearing) {
      float l = norm3(point_G - origin);
      l = std::min(std::max(l - trunc, 0.0f), max_ray);
      b = origin + u * l;
      a = carving ? origin : b;
    } else {
      b = point_G + u * trunc;
      a = carving ? origin : (point_G - u * trunc);
    }
    const V3 as = a * inv, bs = b * inv;
    if (from_origin) {
      setup(as, bs);
    } else {
      setup(bs, as);
    }
  }

  void setup(V3 s, V3 e) {
    if (std::isnan(s.x) || std::isnan(s.y) || std::isnan(s.z) || std::isnan(e.x) || std::isnan(e.y) ||
        std::isnan(e.z)) {
      // the reference leaves current_step_ uninitialised here (integrator_utils.cc:129-134);
      // the restatement defines the ray as empty.
      dead = true;
      return;
    }
    cur = gridIndexScaled(s);
    const L3 end = gridIndexScaled(e);
    len = static_cast<unsigned int>(std::abs(end.x - cur.x) + std::abs(end.y - cur.y) +
                                    std::abs(end.z - cur.z));
    const float r[3] = {e.x - s.x, e.y - s.y, e.z - s.z};
    const float sh[3] = {s.x - static_cast<float>(cur.x), s.y - static_cast<float>(cur.y),
                         s.z - static_cast<float>(cur.z)};
    for (int k = 0; k < 3; ++k) {
      sgn[k] = signumf(r[k]);
      const int corrected = std::max(0, sgn[k]);
      const float to_boundary = static_cast<float>(corrected) - sh[k];
      // the "std::abs(r) < 0.0 ? 2.0 :" guards in the reference are dead code
      tnext[k] = to_boundary / r[k];
      tstep[k] = static_cast<float>(sgn[k]) / r[k];
    }
  }

  bool next(L3* out) {
    if (dead) return false;
    if (step++ > len) return false;
    *out = cur;
    int k = 0;  // first minimum, strict < (Eigen minCoeff visitor)
    float m = tnext[0];
    if (tnext[1] < m) {
      m = tnext[1];
      k = 1;
    }
    if (tnext[2] < m) {
      k = 2;
    }
    (k == 0 ? cur.x : (k == 1 ? cur.y : cur.z)) += sgn[k];
    tnext[k] += tstep[k];
    return true;
  }
};

// ApproxHashSet<20, 10000, GlobalIndex, LongIndexHash> (utils/approx_hash_array.h:75-179)
struct ApproxSet {
  static constexpr size_t kBits = 20, kResetThreshold = 10000;
  size_t offset = 0;
  std::vector<size_t> slots;
  ApproxSet() : slots((size_t(1) << kBits) + kResetThreshold, 0) { slots[0] = std::numeric_limits<size_t>::max(); }
  bool replaceHash(const L3& idx) {
    const size_t h = HashL3()(idx);
    size_t& s = slots[(h & ((size_t(1) << kBits) - 1)) + offset];
    if (s == h) return false;
    s = h;
    return true;
  }
  void reset() {
    if (++offset >= kResetThreshold) {
      std::fill(slots.begin(), slots.end(), 0);
      offset = 0;
      slots[0] = std::numeric_limits<size_t>::max();
    }
  }
};

// utils/bucket_queue.h:18-100
struct BucketQ {
  int nb = 0;
  double maxv = 0;
  std::vector<std::queue<L3>> b;
  int last = 0;
  size_t count = 0;
  void configure(int n, double m) {
    maxv = m;
    nb = n;
    b.clear();
    b.resize(n);
    count = 0;
  }
  void push(const L3& k, double v) {
    if (v > maxv) v = maxv;
    int bi = static_cast<int>(std::floor(std::abs(v) / maxv * (nb - 1)));
    if (bi >= nb) bi = nb - 1;
    if (bi < last) last = bi;
    b[bi].push(k);
    ++count;
  }
  bool empty() const { return count == 0; }
  L3 front() {
    while (b[last].empty() && last < nb) ++last;
    return b[last].front();
  }
  void pop() {
    if (empty()) return;
    while (b[last].empty() && last < nb) ++last;
    if (last < nb) {
      b[last].pop();
      --count;
    }
  }
  void clear() {
    b.clear();
    b.resize(nb);
    last = 0;
    count = 0;
  }
};

// src/utils/neighbor_tools.cc:8-30: 6 faces, 12 edges, 8 corners, in this order
const int kOff[26][3] = {{-1, 0, 0},  {1, 0, 0},   {0, -1, 0},  {0, 1, 0},  {0, 0, -1},  {0, 0, 1},
                         {-1, -1, 0}, {-1, 1, 0},  {1, -1, 0},  {1, 1, 0},  {0, -1, -1}, {0, -1, 1},
                         {0, 1, -1},  {0, 1, 1},   {-1, 0, -1}, {1, 0, -1}, {-1, 0, 1},  {1, 0, 1},
                         {-1, -1, -1}, {-1, -1, 1}, {-1, 1, -1}, {-1, 1, 1}, {1, -1, -1}, {1, -1, 1},
                         {1, 1, -1},  {1, 1, 1}};
inline float nbrDist(int i) {
  static const float s2 = std::sqrt(2), s3 = std::sqrt(3);  // float(sqrt(double))
  return i < 6 ? 1.0f : (i < 18 ? s2 : s3);
}

int64_t g_fast_reset_counter = 0;  // the reference's function-static (tsdf_integrator.cc:564)

// ------------------------------------------------------------------------- the map
struct Map {
  vbo_tsdf_config cfg;
  float voxel_size, voxel_size_inv, block_size, vps_inv;
  int vps;
  BlockMap<TsdfVox> tsdf, temp;
  BlockMap<EsdfVox> esdf;
  ApproxSet start_set, observed_set;
  // esdf state (integrator/esdf_integrator.h:156-178)
  bool has_esdf = false;
  vbo_esdf_config ecfg;
  BucketQ open;
  std::queue<L3> raise;
  std::unordered_set<I3, HashI3> updated_blocks;
  // MeshLayer (mesh/mesh_layer.h:22-310): block index -> Mesh (mesh/mesh.h:36-164)
  struct MeshBlk {
    std::vector<V3> vertices, normals;
    std::vector<Rgba> colors;
    bool updated = false;
  };
  std::unordered_map<I3, MeshBlk, HashI3> mesh;
  // bookkeeping
  double last_seconds = 0;
  uint64_t counters[8] = {0};
  std::unordered_map<I3, std::vector<uint64_t>, HashI3> touched;  // per-scan bitmaps

  Map(const vbo_tsdf_config& c, float vs, int n) : cfg(c), voxel_size(vs), vps(n) {
    // Layer ctor (core/layer.h:36-47) and TsdfIntegratorBase::setLayer (tsdf_integrator.cc:68-80)
    voxel_size_inv = static_cast<float>(1.0 / voxel_size);
    block_size = voxel_size * vps;
    vps_inv = static_cast<float>(1.0 / static_cast<size_t>(vps));
    if (cfg.integrator_threads == 0) cfg.integrator_threads = 1;
    if (cfg.allow_clear && !cfg.voxel_carving_enabled) cfg.allow_clear = 0;  // cc:61-64
  }

  // tsdf_integrator.h:112-129
  bool pointValid(V3 p, bool freespace, bool* clearing) const {
    const float r = norm3(p);
    if (r < cfg.min_ray_length_m) return false;
    if (r > cfg.max_ray_length_m) {
      if (cfg.allow_clear || freespace) {
        *clearing = true;
        return true;
      }
      return false;
    }
    *clearing = freespace;
    return true;
  }
  // tsdf_integrator.cc:231-240
  float pointWeight(V3 p) const {
    if (cfg.use_const_weight) return 1.0f;
    const float z = std::abs(p.z);
    return z > kEps ? 1.0f / (z * z) : 0.0f;
  }

  // tsdf_integrator.cc:91-134: layer lookup, else the temporary block map; sets all updated bits
  TsdfVox* voxelFor(const L3& g) {
    const I3 bi = blockOf(g, vps_inv);
    std::shared_ptr<Blk<TsdfVox>> blk;
    auto it = tsdf.find(bi);
    if (it != tsdf.end()) {
      blk = it->second;
    } else {
      auto jt = temp.find(bi);
      if (jt != temp.end()) {
        blk = jt->second;
      } else {
        blk = temp.emplace(bi, std::make_shared<Blk<TsdfVox>>(vps)).first->second;
        ++counters[5];
      }
    }
    blk->updated = 7;
    const size_t lin = localLinear(g, vps);
    std::vector<uint64_t>& bits = touched[bi];
    if (bits.empty()) bits.assign((static_cast<size_t>(vps) * vps * vps + 63) / 64, 0);
    bits[lin >> 6] |= uint64_t(1) << (lin & 63);
    return &blk->vox[lin];
  }
  // tsdf_integrator.cc:137-147
  void commitTemp() {
    for (const auto& kv : temp) tsdf.insert(kv);
    temp.clear();
  }

  // tsdf_integrator.cc:150-209 (+ computeDistance :216-228)
  void updateVoxel(V3 origin, V3 point_G, const L3& g, Rgba color, float weight, TsdfVox* v) {
    ++counters[2];
    const V3 c = centerPoint(g, voxel_size);
    const V3 vo = c - origin, po = point_G - origin;
    const float dist_G = norm3(po);
    const float dist_G_V = dot3(vo, po) / dist_G;
    const float sdf = dist_G - dist_G_V;
    const float T = cfg.default_truncation_distance;
    float w = weight;
    const float eps = voxel_size;
    if (cfg.use_weight_dropoff && sdf < -eps) {
      w = weight * (T + sdf) / (T - eps);
      w = std::max(w, 0.0f);
    }
    if (cfg.use_sparsity_compensation_factor) {
      if (std::abs(sdf) < T) w *= cfg.sparsity_compensation_factor;
    }
    const float new_w = v->weight + w;
    if (new_w < kEps) return;
    const float new_sdf = (sdf * w + v->distance * v->weight) / new_w;
    if (std::abs(sdf) < T) v->color = blend(v->color, v->weight, color, w);
    v->distance = (new_sdf > 0.0) ? std::min(T, new_sdf) : std::max(-T, new_sdf);
    v->weight = std::min(cfg.max_weight, new_w);
  }

  // integrator_utils.cc:17-67: the order in which one thread hands out point indices
  std::vector<size_t> pointOrder(const float* xyz, size_t n) const {
    std::vector<size_t> order(n);
    if (cfg.integration_order_mode == 1) {
      std::vector<std::pair<size_t, double>> v;
      v.reserve(n);
      for (size_t i = 0; i < n; ++i) {
        v.emplace_back(i, sqnorm3(V3{xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2]}));
      }
      std::sort(v.begin(), v.end(),
                [](const std::pair<size_t, double>& a, const std::pair<size_t, double>& b) {
                  return a.second < b.second;
                });
      for (size_t i = 0; i < n; ++i) order[i] = v[i].first;
    } else {
      const size_t groups = n / 1024;
      for (size_t s = 0; s < n; ++s) {
        order[s] = (groups * 1024 <= s) ? s : (s % groups) * 1024 + s / groups;
      }
    }
    return order;
  }

  // SimpleTsdfIntegrator::integrateFunction, tsdf_integrator.cc:269-305
  void integrateSimple(const Pose& T, const float* xyz, const uint8_t* rgba, size_t n, bool freespace) {
    const V3 origin = T.t;
    for (size_t idx : pointOrder(xyz, n)) {
      const V3 p{xyz[3 * idx], xyz[3 * idx + 1], xyz[3 * idx + 2]};
      bool clearing;
      if (!pointValid(p, freespace, &clearing)) continue;
      ++counters[6];
      ++counters[clearing ? 1 : 0];
      const V3 pg = T.apply(p);
      const Rgba col{rgba[4 * idx], rgba[4 * idx + 1], rgba[4 * idx + 2], rgba[4 * idx + 3]};
      Dda dda(origin, pg, clearing, cfg.voxel_carving_enabled, cfg.max_ray_length_m, voxel_size_inv,
              cfg.default_truncation_distance, true);
      L3 g;
      while (dda.next(&g)) {
        TsdfVox* v = voxelFor(g);
        updateVoxel(origin, pg, g, col, pointWeight(p), v);
      }
    }
    commitTemp();
  }

  // MergedTsdfIntegrator, tsdf_integrator.cc:307-486
  typedef std::unordered_map<L3, std::vector<size_t>, HashL3> BundleMap;

  void castBundle(const Pose& T, const float* xyz, const uint8_t* rgba, bool clearing, const L3& key,
                  const std::vector<size_t>& members, const BundleMap& voxel_map) {
    if (members.empty()) return;
    const V3 origin = T.t;
    Rgba mcol{0, 0, 0, 0};
    V3 mp{0, 0, 0};
    float mw = 0.0f;
    for (size_t idx : members) {  // cc:387-405: running weighted mean in the camera frame
      const V3 p{xyz[3 * idx], xyz[3 * idx + 1], xyz[3 * idx + 2]};
      const float w = pointWeight(p);
      if (w < kEps) continue;
      mp = (mp * mw + p * w) / (mw + w);
      mcol = blend(mcol, mw, Rgba{rgba[4 * idx], rgba[4 * idx + 1], rgba[4 * idx + 2], rgba[4 * idx + 3]}, w);
      mw += w;
      if (clearing) break;
    }
    const V3 pg = T.apply(mp);
    ++counters[clearing ? 1 : 0];
    Dda dda(origin, pg, clearing, cfg.voxel_carving_enabled, cfg.max_ray_length_m, voxel_size_inv,
            cfg.default_truncation_distance, true);
    L3 g;
    while (dda.next(&g)) {
      if (cfg.enable_anti_grazing) {  // cc:415-422
        if ((clearing || g != key) && voxel_map.find(g) != voxel_map.end()) continue;
      }
      TsdfVox* v = voxelFor(g);
      updateVoxel(origin, pg, g, mcol, mw, v);
    }
  }

  void integrateMerged(const Pose& T, const float* xyz, const uint8_t* rgba, size_t n, bool freespace) {
    BundleMap voxel_map, clear_map;
    for (size_t idx : pointOrder(xyz, n)) {  // bundleRays, cc:340-371
      const V3 p{xyz[3 * idx], xyz[3 * idx + 1], xyz[3 * idx + 2]};
      bool clearing;
      if (!pointValid(p, freespace, &clearing)) continue;
      ++counters[6];
      const L3 key = gridIndex(T.apply(p), voxel_size_inv);
      (clearing ? clear_map : voxel_map)[key].push_back(idx);
    }
    for (int pass = 0; pass < 2; ++pass) {  // integrateRays(false) then (true), cc:323-335
      const BundleMap& m = pass ? clear_map : voxel_map;
      // one thread visits every map entry in iteration order (cc:434-457 with threads == 1)
      for (const auto& kv : m) castBundle(T, xyz, rgba, pass == 1, kv.first, kv.second, voxel_map);
      commitTemp();  // cc:482-485
    }
  }

  // FastTsdfIntegrator, tsdf_integrator.cc:488-590
  void integrateFast(const Pose& T, const float* xyz, const uint8_t* rgba, size_t n, bool freespace) {
    const auto start = std::chrono::steady_clock::now();
    if ((++g_fast_reset_counter) >= cfg.clear_checks_every_n_frames) {
      g_fast_reset_counter = 0;
      start_set.reset();
      observed_set.reset();
    }
    const V3 origin = T.t;
    for (size_t idx : pointOrder(xyz, n)) {
      if (!(std::chrono::duration_cast<std::chrono::microseconds>(std::chrono::steady_clock::now() - start)
                .count() < cfg.max_integration_time_s * 1000000)) {
        break;
      }
      const V3 p{xyz[3 * idx], xyz[3 * idx + 1], xyz[3 * idx + 2]};
      bool clearing;
      if (!pointValid(p, freespace, &clearing)) continue;
      ++counters[6];
      const V3 pg = T.apply(p);
      L3 g = gridIndex(pg, cfg.start_voxel_subsampling_factor * voxel_size_inv);
      if (!start_set.replaceHash(g)) continue;
      ++counters[clearing ? 1 : 0];
      const Rgba col{rgba[4 * idx], rgba[4 * idx + 1], rgba[4 * idx + 2], rgba[4 * idx + 3]};
      Dda dda(origin, pg, clearing, cfg.voxel_carving_enabled, cfg.max_ray_length_m, voxel_size_inv,
              cfg.default_truncation_distance, false);
      int64_t collisions = 0;
      while (dda.next(&g)) {
        if (!observed_set.replaceHash(g)) {
          ++collisions;
        } else {
          collisions = 0;
        }
        if (collisions > cfg.max_consecutive_ray_collisions) break;
        TsdfVox* v = voxelFor(g);
        updateVoxel(origin, pg, g, col, pointWeight(p), v);
      }
    }
    commitTemp();
  }

  // --------------------------------------------------------------------------- ESDF
  EsdfVox* esdfVoxel(const L3& g) {  // Layer::getVoxelPtrByGlobalIndex, core/layer.h:228-239
    auto it = esdf.find(blockOf(g, vps_inv));
    if (it == esdf.end()) return nullptr;
    return &it->second->vox[localLinear(g, vps)];
  }
  std::shared_ptr<Blk<EsdfVox>> esdfAllocate(const I3& bi) {  // core/layer.h:103-111
    auto it = esdf.find(bi);
    if (it != esdf.end()) return it->second;
    return esdf.emplace(bi, std::make_shared<Blk<EsdfVox>>(vps)).first->second;
  }
  bool isFixed(float d) const { return std::abs(d) < ecfg.min_distance_m; }  // esdf_integrator.h:131-133

  // esdf_integrator.cc:498-530 (note: neighbour distance in VOXELS, cc:508)
  bool updateFromNeighbors(const L3& g) {
    EsdfVox* v = esdfVoxel(g);
    for (int i = 0; i < 26; ++i) {
      const L3 ng{g.x + kOff[i][0], g.y + kOff[i][1], g.z + kOff[i][2]};
      EsdfVox* nv = esdfVoxel(ng);
      if (nv == nullptr) continue;
      if (!nv->observed || nv->distance >= ecfg.max_distance_m || nv->distance <= -ecfg.max_distance_m) continue;
      if (signumf(nv->distance) == signumf(v->distance)) {
        if (std::abs(nv->distance) < std::abs(v->distance)) {
          v->distance = nv->distance + signumf(v->distance) * nbrDist(i);
          v->parent[0] = -kOff[i][0];
          v->parent[1] = -kOff[i][1];
          v->parent[2] = -kOff[i][2];
          return true;
        }
      }
    }
    return false;
  }

  // esdf_integrator.cc:124-302
  void esdfFromBlocks(const std::vector<I3>& blocks, bool incremental) {
    const float dflt = ecfg.default_distance_m, md = ecfg.min_diff_m;
    for (const I3& bi : blocks) {
      auto tb = tsdf.find(bi);
      if (tb == tsdf.end()) continue;
      std::shared_ptr<Blk<EsdfVox>> eb = esdfAllocate(bi);
      eb->updated = 1;  // set_updated(true): bitset(1ull) => only kMap (cc:147)
      const size_t nv = tb->second->vox.size();
      for (size_t lin = 0; lin < nv; ++lin) {
        const TsdfVox& tv = tb->second->vox[lin];
        if (tv.weight < ecfg.min_weight) {
          if (!incremental && ecfg.add_occupied_crust) {
            EsdfVox& ev = eb->vox[lin];
            ev.distance = -dflt;
            ev.observed = 1;
            ev.hallucinated = 1;
            ev.fixed = 0;
          }
          continue;
        }
        EsdfVox& ev = eb->vox[lin];
        const int z = static_cast<int>(lin) / (vps * vps), rem = static_cast<int>(lin) % (vps * vps);
        const L3 g{int64_t(bi.x) * vps + rem % vps, int64_t(bi.y) * vps + rem / vps, int64_t(bi.z) * vps + z};
        const bool tfixed = isFixed(tv.distance);
        if (!ev.observed || ev.hallucinated) {
          if (ev.hallucinated) raise.push(g);
          if (tfixed) {
            ev.distance = tv.distance;
            ev.fixed = 1;
            ev.in_queue = 1;
            open.push(g, ev.distance);
          } else {
            ev.distance = signumf(tv.distance) * dflt;
            ev.fixed = 0;
            if (incremental) {
              if (updateFromNeighbors(g)) {
                ev.in_queue = 1;
                open.push(g, ev.distance);
              }
            }
          }
          ev.parent[0] = ev.parent[1] = ev.parent[2] = 0;
        } else {
          if (tfixed || ev.fixed) {
            if (!tfixed) {
              ev.distance = signumf(tv.distance) * dflt;
              ev.parent[0] = ev.parent[1] = ev.parent[2] = 0;
              ev.fixed = 0;
              raise.push(g);
              ev.in_queue = 1;
              open.push(g, ev.distance);
            } else if ((ev.distance > 0.0f && tv.distance + md < ev.distance) ||
                       (ev.distance <= 0.0f && tv.distance - md > ev.distance)) {
              ev.fixed = tfixed;
              ev.distance = ev.fixed ? tv.distance : signumf(tv.distance) * dflt;
              ev.parent[0] = ev.parent[1] = ev.parent[2] = 0;
              ev.in_queue = 1;
              open.push(g, ev.distance);
            } else if ((ev.distance > 0.0f && tv.distance - md > ev.distance) ||
                       (ev.distance <= 0.0f && tv.distance + md < ev.distance)) {
              ev.fixed = tfixed;
              ev.distance = ev.fixed ? tv.distance : signumf(tv.distance) * dflt;
              ev.parent[0] = ev.parent[1] = ev.parent[2] = 0;
              raise.push(g);
              ev.in_queue = 1;
              open.push(g, ev.distance);
            }
          } else if (signumf(tv.distance) != signumf(ev.distance)) {
            if (tv.distance < ev.distance) {
              ev.distance = signumf(tv.distance) * dflt;
              ev.parent[0] = ev.parent[1] = ev.parent[2] = 0;
              ev.in_queue = 1;
              open.push(g, ev.distance);
            } else {
              ev.distance = signumf(tv.distance) * dflt;
              ev.parent[0] = ev.parent[1] = ev.parent[2] = 0;
              raise.push(g);
            }
          }
        }
        ev.observed = 1;
        ev.hallucinated = 0;
      }
    }
    processRaise();
    processOpen();
  }

  // esdf_integrator.cc:305-369
  void processRaise() {
    while (!raise.empty()) {
      const L3 g = raise.front();
      raise.pop();
      for (int i = 0; i < 26; ++i) {
        const L3 ng{g.x + kOff[i][0], g.y + kOff[i][1], g.z + kOff[i][2]};
        EsdfVox* nv = esdfVoxel(ng);
        if (nv == nullptr) continue;
        if (!nv->observed || nv->fixed) continue;
        bool is_parent = nv->parent[0] == -kOff[i][0] && nv->parent[1] == -kOff[i][1] &&
                         nv->parent[2] == -kOff[i][2];
        if (ecfg.full_euclidean_distance) {
          V3 pd = unit3(V3{float(nv->parent[0]), float(nv->parent[1]), float(nv->parent[2])});
          is_parent = static_cast<int>(std::round(pd.x)) == -kOff[i][0] &&
                      static_cast<int>(std::round(pd.y)) == -kOff[i][1] &&
                      static_cast<int>(std::round(pd.z)) == -kOff[i][2];
        }
        if (is_parent) {
          nv->distance = signumf(nv->distance) * ecfg.default_distance_m;
          nv->parent[0] = nv->parent[1] = nv->parent[2] = 0;
          raise.push(ng);
        } else if (!nv->in_queue) {
          open.push(ng, nv->distance);
          nv->in_queue = 1;
        }
      }
    }
  }

  // esdf_integrator.cc:371-496
  void processOpen() {
    const float md = ecfg.min_diff_m;
    while (!open.empty()) {
      const L3 g = open.front();
      open.pop();
      EsdfVox* v = esdfVoxel(g);
      v->in_queue = 0;
      if (!v->observed || v->distance >= ecfg.max_distance_m || v->distance <= -ecfg.max_distance_m) continue;
      for (int i = 0; i < 26; ++i) {
        const L3 ng{g.x + kOff[i][0], g.y + kOff[i][1], g.z + kOff[i][2]};
        float dist = nbrDist(i) * voxel_size;
        EsdfVox* nv = esdfVoxel(ng);
        if (nv == nullptr) continue;
        if (!nv->observed || nv->fixed) continue;
        int np[3] = {-kOff[i][0], -kOff[i][1], -kOff[i][2]};
        if (ecfg.full_euclidean_distance) {
          np[0] = v->parent[0] - kOff[i][0];
          np[1] = v->parent[1] - kOff[i][1];
          np[2] = v->parent[2] - kOff[i][2];
          dist = voxel_size * (norm3(V3{float(np[0]), float(np[1]), float(np[2])}) -
                               norm3(V3{float(v->parent[0]), float(v->parent[1]), float(v->parent[2])}));
          if (dist < 0.0) continue;
        }
        bool changed = false;
        if (v->distance > 0 && nv->distance > 0) {
          if (v->distance + dist + md < nv->distance) {
            nv->distance = v->distance + dist;
            changed = true;
          }
        } else if (v->distance <= 0 && nv->distance <= 0) {
          if (v->distance - dist - md > nv->distance) {
            nv->distance = v->distance - dist;
            changed = true;
          }
        } else {
          const float pot = v->distance - signumf(v->distance) * dist;
          if (std::abs(pot - nv->distance) > dist) {
            if (signumf(pot) == nv->distance) {  // sic (cc:464): a sign compared with a distance
              nv->distance = pot;
            } else {
              nv->distance = signumf(nv->distance) * dist;
            }
            changed = true;
          }
        }
        if (changed) {
          nv->parent[0] = np[0];
          nv->parent[1] = np[1];
          nv->parent[2] = np[2];
          if (ecfg.multi_queue || !nv->in_queue) {
            open.push(ng, nv->distance);
            nv->in_queue = 1;
          }
        }
      }
    }
  }

  // esdf_integrator.cc:94-122
  void esdfUpdate(bool batch, bool clear_flag) {
    std::vector<I3> blocks;
    if (batch) {
      esdf.clear();
      for (const auto& kv : tsdf) blocks.push_back(kv.first);
    } else {
      for (const auto& kv : tsdf) {
        if (kv.second->updated & 4) blocks.push_back(kv.first);
      }
    }
    blocks.insert(blocks.end(), updated_blocks.begin(), updated_blocks.end());
    updated_blocks.clear();
    esdfFromBlocks(blocks, !batch);
    if (!batch && clear_flag) {
      for (const I3& bi : blocks) {
        auto it = tsdf.find(bi);
        if (it != tsdf.end()) it->second->updated &= static_cast<uint8_t>(~4);
      }
    }
  }

  // ------------------------------------------------------------------ meshing
  // Block::computeCoordinatesFromVoxelIndex (core/block.h:90-92): origin_ + centre, with
  // origin_ = float(block index) * block_size (core/common.h:196-201, core/layer.h:133-140)
  V3 blockOrigin(const I3& bi) const {
    return V3{static_cast<float>(bi.x) * block_size, static_cast<float>(bi.y) * block_size,
              static_cast<float>(bi.z) * block_size};
  }
  // utils/meshing_utils.h:16-24
  static bool sdfIfValid(const TsdfVox& v, float min_weight, float* sdf) {
    if (v.weight <= min_weight) return false;
    *sdf = v.distance;
    return true;
  }
  // mesh/marching_cubes.h:150-164
  static V3 interpolateVertex(V3 v1, V3 v2, float sdf1, float sdf2) {
    const float kMinSdfDifference = 1e-6f;
    const float diff = sdf1 - sdf2;
    if (std::abs(diff) >= kMinSdfDifference) {
      const float t = sdf1 / diff;
      return v1 + (v2 - v1) * t;
    }
    return (v1 + v2) * 0.5f;
  }
  // mesh/marching_cubes.h:74-113 (the Mesh overload) with :115-147
  static void meshCube(const V3 corner[8], const float sdf[8], MeshBlk* out) {
    static const uint64_t kTri[256] = {VBX_MC_TRIANGLE_WORDS};
    static const int kPairs[12][2] = {VBX_MC_EDGE_PAIRS};
    int index = 0;
    for (int i = 0; i < 8; ++i) index |= (sdf[i] < 0 ? (1 << i) : 0);
    if (index == 0) return;
    V3 edge[12];
    for (int i = 0; i < 12; ++i) {
      const int a = kPairs[i][0], b = kPairs[i][1];
      if ((sdf[a] < 0 && sdf[b] >= 0) || (sdf[a] >= 0 && sdf[b] < 0)) {
        edge[i] = interpolateVertex(corner[a], corner[b], sdf[a], sdf[b]);
      }
    }
    const uint64_t row = kTri[index];
    for (int col = 0; col < 15 && ((row >> (4 * col)) & 0xF) != 0xF; col += 3) {
      const V3 p0 = edge[(row >> (4 * (col + 2))) & 0xF];
      const V3 p1 = edge[(row >> (4 * (col + 1))) & 0xF];
      const V3 p2 = edge[(row >> (4 * col)) & 0xF];
      out->vertices.push_back(p0);
      out->vertices.push_back(p1);
      out->vertices.push_back(p2);
      const V3 n = unit3(cross3(p1 - p0, p2 - p0));
      out->normals.push_back(n);
      out->normals.push_back(n);
      out->normals.push_back(n);
    }
  }
  // mesh_integrator.h:262-290 (inside) and :292-366 (border): the cube whose lowest corner is voxel
  // `vi` of block `bi`; corners outside the block come from the neighbouring blocks
  void meshOneCube(const I3& bi, const Blk<TsdfVox>& blk, const I3& vi, float min_weight, MeshBlk* out) const {
    static const int kOff[8][3] = {{0, 0, 0}, {1, 0, 0}, {1, 1, 0}, {0, 1, 0},
                                   {0, 0, 1}, {1, 0, 1}, {1, 1, 1}, {0, 1, 1}};  // cube_index_offsets_, :94-95
    const V3 coords = blockOrigin(bi) + centerPoint(L3{vi.x, vi.y, vi.z}, voxel_size);
    V3 corner[8];
    float sdf[8];
    for (int i = 0; i < 8; ++i) {
      int cx = vi.x + kOff[i][0], cy = vi.y + kOff[i][1], cz = vi.z + kOff[i][2];
      const Blk<TsdfVox>* src = &blk;
      if (cx >= vps || cy >= vps || cz >= vps) {
        I3 nb = bi;
        if (cx >= vps) {
          nb.x += 1;
          cx -= vps;
        }
        if (cy >= vps) {
          nb.y += 1;
          cy -= vps;
        }
        if (cz >= vps) {
          nb.z += 1;
          cz -= vps;
        }
        auto it = tsdf.find(nb);
        if (it == tsdf.end()) return;  // all_neighbors_observed = false, :358-361
        src = it->second.get();
      }
      if (!sdfIfValid(src->vox[cx + vps * (cy + cz * vps)], min_weight, &sdf[i])) return;
      const V3 off{static_cast<float>(kOff[i][0]) * voxel_size, static_cast<float>(kOff[i][1]) * voxel_size,
                   static_cast<float>(kOff[i][2]) * voxel_size};
      corner[i] = coords + off;
    }
    meshCube(corner, sdf, out);
  }
  // mesh_integrator.h:368-388
  void meshColors(const I3& bi, const Blk<TsdfVox>& blk, float min_weight, MeshBlk* out) const {
    out->colors.assign(out->vertices.size(), Rgba{0, 0, 0, 0});
    const V3 origin = blockOrigin(bi);
    const float block_size_inv = static_cast<float>(1.0 / block_size);
    for (size_t i = 0; i < out->vertices.size(); ++i) {
      const V3 v = out->vertices[i];
      const L3 vi = gridIndex(v - origin, voxel_size_inv);  // computeVoxelIndexFromCoordinates, core/block.h:65-70
      const TsdfVox* vox = nullptr;
      if (vi.x >= 0 && vi.x < vps && vi.y >= 0 && vi.y < vps && vi.z >= 0 && vi.z < vps) {
        vox = &blk.vox[vi.x + vps * (vi.y + vi.z * vps)];
      } else {
        const L3 nbl = gridIndex(v, block_size_inv);  // Layer::computeBlockIndexFromCoordinates, core/layer.h:128-131
        const I3 nb{static_cast<int>(nbl.x), static_cast<int>(nbl.y), static_cast<int>(nbl.z)};
        auto it = tsdf.find(nb);
        if (it == tsdf.end()) continue;  // (the reference dereferences a null block pointer here)
        // Block::getVoxelByCoordinates -> computeTruncatedVoxelIndexFromCoordinates, core/block_inl.h:29-40
        const L3 t = gridIndex(v - blockOrigin(nb), voxel_size_inv);
        const int64_t mx = vps - 1;
        const int64_t tx = std::max<int64_t>(std::min(t.x, mx), 0), ty = std::max<int64_t>(std::min(t.y, mx), 0),
                      tz = std::max<int64_t>(std::min(t.z, mx), 0);
        vox = &it->second->vox[tx + vps * (ty + tz * vps)];
      }
      if (vox->weight > min_weight) out->colors[i] = vox->color;  // utils/meshing_utils.h:45-54
    }
  }
  // MeshIntegrator::generateMesh (mesh_integrator.h:132-160) + updateMeshForBlock (:238-260) +
  // extractBlockMesh (:179-236, the cube order of the four loops)
  void generateMesh(bool use_color, float min_weight, bool only_updated, bool clear_flag) {
    std::vector<I3> blocks;
    for (const auto& kv : tsdf) {
      if (!only_updated || (kv.second->updated & 2)) blocks.push_back(kv.first);
    }
    for (const I3& bi : blocks) {
      MeshBlk& mb = mesh[bi];  // allocateMeshPtrByIndex
      mb.vertices.clear();
      mb.normals.clear();
      mb.colors.clear();
      Blk<TsdfVox>& blk = *tsdf.find(bi)->second;
      I3 vi;
      for (vi.x = 0; vi.x < vps - 1; ++vi.x) {
        for (vi.y = 0; vi.y < vps - 1; ++vi.y) {
          for (vi.z = 0; vi.z < vps - 1; ++vi.z) meshOneCube(bi, blk, vi, min_weight, &mb);
        }
      }
      vi.x = vps - 1;  // max X plane
      for (vi.z = 0; vi.z < vps; ++vi.z) {
        for (vi.y = 0; vi.y < vps; ++vi.y) meshOneCube(bi, blk, vi, min_weight, &mb);
      }
      vi.y = vps - 1;  // max Y plane
      for (vi.z = 0; vi.z < vps; ++vi.z) {
        for (vi.x = 0; vi.x < vps - 1; ++vi.x) meshOneCube(bi, blk, vi, min_weight, &mb);
      }
      vi.z = vps - 1;  // max Z plane
      for (vi.y = 0; vi.y < vps - 1; ++vi.y) {
        for (vi.x = 0; vi.x < vps - 1; ++vi.x) meshOneCube(bi, blk, vi, min_weight, &mb);
      }
      if (use_color) meshColors(bi, blk, min_weight, &mb);
      mb.updated = true;
      if (clear_flag) blk.updated &= static_cast<uint8_t>(~2);  // updated().reset(Update::kMesh), :171-175
    }
  }

  // utils/planning_utils_inl.h:15-62 + esdf_integrator.cc:25-92
  typedef std::unordered_map<I3, std::vector<I3>, HashI3> HierMap;
  void sphereAround(V3 center, float radius, HierMap* out) {
    const float inv = static_cast<float>(1.0 / voxel_size);
    const L3 c = gridIndex(center, inv);
    const float rv = radius / voxel_size;
    for (float x = -rv; x <= rv; x++) {
      for (float y = -rv; y <= rv; y++) {
        for (float z = -rv; z <= rv; z++) {
          if (norm3(V3{x, y, z}) <= rv) {
            const L3 g{static_cast<int64_t>(std::floor(x)) + c.x, static_cast<int64_t>(std::floor(y)) + c.y,
                       static_cast<int64_t>(std::floor(z)) + c.z};
            const I3 bi = blockOf(g, static_cast<float>(1.0 / vps));
            constexpr int64_t off = int64_t(1) << 31;
            (*out)[bi].push_back(I3{static_cast<int>((g.x + off) & (vps - 1)), static_cast<int>((g.y + off) & (vps - 1)),
                                    static_cast<int>((g.z + off) & (vps - 1))});
          }
        }
      }
    }
    for (auto& kv : *out) esdfAllocate(kv.first);
  }
  void addRobotPosition(V3 p) {
    HierMap inner;
    sphereAround(p, ecfg.clear_sphere_radius, &inner);
    for (auto& kv : inner) {
      std::shared_ptr<Blk<EsdfVox>> b = esdf.find(kv.first)->second;
      for (const I3& vi : kv.second) {
        EsdfVox& ev = b->vox[vi.x + vps * (vi.y + vi.z * vps)];
        if (!ev.observed || ev.hallucinated) {
          if (ev.hallucinated) {
            raise.push(L3{int64_t(kv.first.x) * vps + vi.x, int64_t(kv.first.y) * vps + vi.y,
                          int64_t(kv.first.z) * vps + vi.z});
          }
          ev.distance = ecfg.default_distance_m;
          ev.observed = 1;
          ev.hallucinated = 1;
          ev.parent[0] = ev.parent[1] = ev.parent[2] = 0;
          updated_blocks.insert(kv.first);
        }
      }
    }
    HierMap outer;
    sphereAround(p, ecfg.occupied_sphere_radius, &outer);
    for (auto& kv : outer) {
      std::shared_ptr<Blk<EsdfVox>> b = esdf.find(kv.first)->second;
      for (const I3& vi : kv.second) {
        EsdfVox& ev = b->vox[vi.x + vps * (vi.y + vi.z * vps)];
        if (!ev.observed) {
          ev.distance = -ecfg.default_distance_m;
          ev.observed = 1;
          ev.hallucinated = 1;
          ev.parent[0] = ev.parent[1] = ev.parent[2] = 0;
          updated_blocks.insert(kv.first);
        } else if (!ev.in_queue) {
          open.push(L3{int64_t(kv.first.x) * vps + vi.x, int64_t(kv.first.y) * vps + vi.y,
                       int64_t(kv.first.z) * vps + vi.z},
                    ev.distance);
        }
      }
    }
  }
};

template <typename V>
void sortedKeys(const BlockMap<V>& m, int32_t* out) {
  std::vector<I3> k;
  k.reserve(m.size());
  for (const auto& kv : m) k.push_back(kv.first);
  std::sort(k.begin(), k.end(), [](const I3& a, const I3& b) {
    if (a.x != b.x) return a.x < b.x;
    if (a.y != b.y) return a.y < b.y;
    return a.z < b.z;
  });
  for (size_t i = 0; i < k.size(); ++i) {
    out[3 * i] = k[i].x;
    out[3 * i + 1] = k[i].y;
    out[3 * i + 2] = k[i].z;
  }
}

}  // namespace

extern "C" {

const char* vbo_impl_name(void) { return "port"; }

void* vbo_create(const vbo_tsdf_config* c, float voxel_size, int voxels_per_side) {
  return new Map(*c, voxel_size, voxels_per_side);
}
void vbo_destroy(void* h) { delete static_cast<Map*>(h); }

int vbo_integrate(void* hv, int kind, const float q[4], const float t[3], const float* xyz,
                  const uint8_t* rgba, uint64_t n, int freespace, int bundle_order) {
  Map* m = static_cast<Map*>(hv);
  if (kind < 1 || kind > 3) return 2;
  const Pose T{q[0], q[1], q[2], q[3], V3{t[0], t[1], t[2]}};
  std::memset(m->counters, 0, sizeof(m->counters));
  m->touched.clear();
  const auto t0 = std::chrono::steady_clock::now();
  if (kind == VBO_SIMPLE) {
    m->integrateSimple(T, xyz, rgba, n, freespace != 0);
  } else if (kind == VBO_MERGED) {
    if (bundle_order != VBO_ORDER_REFERENCE) return 3;  // one order: the reference's
    m->integrateMerged(T, xyz, rgba, n, freespace != 0);
  } else {
    m->integrateFast(T, xyz, rgba, n, freespace != 0);
  }
  m->last_seconds = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
  uint64_t u = 0;
  for (const auto& kv : m->touched) {
    for (uint64_t w : kv.second) u += static_cast<uint64_t>(__builtin_popcountll(w));
  }
  m->counters[3] = u;
  m->counters[4] = m->touched.size();
  return 0;
}

double vbo_last_seconds(void* h) { return static_cast<Map*>(h)->last_seconds; }
void vbo_last_counters(void* h, uint64_t out[8]) {
  std::memcpy(out, static_cast<Map*>(h)->counters, 8 * sizeof(uint64_t));
}

uint64_t vbo_num_blocks(void* hv, int layer) {
  Map* m = static_cast<Map*>(hv);
  return layer == VBO_LAYER_TSDF ? m->tsdf.size() : m->esdf.size();
}
void vbo_block_indices(void* hv, int layer, int32_t* out) {
  Map* m = static_cast<Map*>(hv);
  if (layer == VBO_LAYER_TSDF) {
    sortedKeys(m->tsdf, out);
  } else {
    sortedKeys(m->esdf, out);
  }
}
int vbo_get_block(void* hv, int layer, const int32_t idx[3], void* voxels, uint8_t* updated_bits) {
  Map* m = static_cast<Map*>(hv);
  const I3 bi{idx[0], idx[1], idx[2]};
  if (layer == VBO_LAYER_TSDF) {
    auto it = m->tsdf.find(bi);
    if (it == m->tsdf.end()) return 1;
    std::memcpy(voxels, it->second->vox.data(), it->second->vox.size() * sizeof(TsdfVox));
    if (updated_bits) *updated_bits = it->second->updated;
  } else {
    auto it = m->esdf.find(bi);
    if (it == m->esdf.end()) return 1;
    std::memcpy(voxels, it->second->vox.data(), it->second->vox.size() * sizeof(EsdfVox));
    if (updated_bits) *updated_bits = it->second->updated;
  }
  return 0;
}

// src/core/block.cc:8-41: the int8 fields are ORed in as sign-extended ints, so a negative y or z
// also sets every byte above it
static uint32_t serializeDirection(const int32_t parent[3]) {
  uint32_t data = 0;
  const int8_t px = static_cast<int8_t>(std::min(127, std::max(parent[0], -128)));
  const int8_t py = static_cast<int8_t>(std::min(127, std::max(parent[1], -128)));
  const int8_t pz = static_cast<int8_t>(std::min(127, std::max(parent[2], -128)));
  data |= static_cast<uint32_t>(static_cast<int8_t>(px) << 24);
  data |= static_cast<uint32_t>(static_cast<int8_t>(py) << 16);
  data |= static_cast<uint32_t>(static_cast<int8_t>(pz) << 8);
  return data;
}
int vbo_serialize_block(void* hv, int layer, const int32_t idx[3], uint32_t* words) {
  Map* m = static_cast<Map*>(hv);
  const I3 bi{idx[0], idx[1], idx[2]};
  if (layer == VBO_LAYER_TSDF) {  // block.cc:159-183
    auto it = m->tsdf.find(bi);
    if (it == m->tsdf.end()) return 1;
    for (const TsdfVox& v : it->second->vox) {
      uint32_t w;
      std::memcpy(&w, &v.distance, 4);
      *words++ = w;
      std::memcpy(&w, &v.weight, 4);
      *words++ = w;
      *words++ = static_cast<uint32_t>(v.color.a) | (static_cast<uint32_t>(v.color.b) << 8) |
                 (static_cast<uint32_t>(v.color.g) << 16) | (static_cast<uint32_t>(v.color.r) << 24);
    }
  } else {  // block.cc:203-234
    auto it = m->esdf.find(bi);
    if (it == m->esdf.end()) return 1;
    for (const EsdfVox& v : it->second->vox) {
      uint32_t w;
      std::memcpy(&w, &v.distance, 4);
      *words++ = w;
      uint32_t b2 = serializeDirection(v.parent);
      uint8_t flag = 0;
      flag |= v.observed ? 1 : 0;
      flag |= v.hallucinated ? 2 : 0;
      flag |= v.in_queue ? 4 : 0;
      flag |= v.fixed ? 8 : 0;
      b2 |= static_cast<uint32_t>(flag) & 0xFFu;
      *words++ = b2;
    }
  }
  return 0;
}
int vbo_deserialize_block(void* hv, int layer, const int32_t idx[3], const uint32_t* words) {
  Map* m = static_cast<Map*>(hv);
  const I3 bi{idx[0], idx[1], idx[2]};
  if (layer == VBO_LAYER_TSDF) {  // block.cc:65-90
    auto it = m->tsdf.find(bi);
    if (it == m->tsdf.end()) it = m->tsdf.emplace(bi, std::make_shared<Blk<TsdfVox>>(m->vps)).first;
    for (TsdfVox& v : it->second->vox) {
      std::memcpy(&v.distance, words++, 4);
      std::memcpy(&v.weight, words++, 4);
      const uint32_t b3 = *words++;
      v.color.r = static_cast<uint8_t>(b3 >> 24);
      v.color.g = static_cast<uint8_t>((b3 & 0x00FF0000u) >> 16);
      v.color.b = static_cast<uint8_t>((b3 & 0x0000FF00u) >> 8);
      v.color.a = static_cast<uint8_t>(b3 & 0x000000FFu);
    }
  } else {  // block.cc:110-135, :43-63
    std::shared_ptr<Blk<EsdfVox>> b = m->esdfAllocate(bi);
    for (EsdfVox& v : b->vox) {
      std::memcpy(&v.distance, words++, 4);
      const uint32_t b2 = *words++;
      v.observed = (b2 & 1u) ? 1 : 0;
      v.hallucinated = (b2 & 2u) ? 1 : 0;
      v.in_queue = (b2 & 4u) ? 1 : 0;
      v.fixed = (b2 & 8u) ? 1 : 0;
      v.parent[0] = static_cast<int8_t>((b2 >> 24) & 0xFFu);
      v.parent[1] = static_cast<int8_t>((b2 >> 16) & 0xFFu);
      v.parent[2] = static_cast<int8_t>((b2 >> 8) & 0xFFu);
    }
  }
  return 0;
}

int vbo_esdf_create(void* hv, const vbo_esdf_config* c) {
  Map* m = static_cast<Map*>(hv);
  m->ecfg = *c;
  m->has_esdf = true;
  m->open.configure(c->num_buckets, c->max_distance_m);  // esdf_integrator.cc:21
  m->raise = std::queue<L3>();
  m->updated_blocks.clear();
  return 0;
}
int vbo_esdf_update(void* hv, int batch, int clear_updated_flag) {
  Map* m = static_cast<Map*>(hv);
  if (!m->has_esdf) return 2;
  const auto t0 = std::chrono::steady_clock::now();
  m->esdfUpdate(batch != 0, clear_updated_flag != 0);
  m->last_seconds = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
  return 0;
}
int vbo_esdf_update_blocks(void* hv, const int32_t* idx3, uint64_t n, int incremental) {
  Map* m = static_cast<Map*>(hv);
  if (!m->has_esdf) return 2;
  std::vector<I3> blocks;
  for (uint64_t i = 0; i < n; ++i) blocks.push_back(I3{idx3[3 * i], idx3[3 * i + 1], idx3[3 * i + 2]});
  m->esdfFromBlocks(blocks, incremental != 0);  // esdf_integrator.cc:124-302
  return 0;
}
// esdf_integrator.h:139-149
int vbo_esdf_set_max_distance(void* hv, float max_distance) {
  Map* m = static_cast<Map*>(hv);
  if (!m->has_esdf) return 2;
  m->ecfg.max_distance_m = max_distance;
  if (m->ecfg.default_distance_m < max_distance) m->ecfg.default_distance_m = max_distance;
  return 0;
}
int vbo_esdf_set_full_euclidean(void* hv, int full_euclidean) {
  Map* m = static_cast<Map*>(hv);
  if (!m->has_esdf) return 2;
  m->ecfg.full_euclidean_distance = full_euclidean;
  return 0;
}
int vbo_esdf_add_robot_position(void* hv, const float p[3]) {
  Map* m = static_cast<Map*>(hv);
  if (!m->has_esdf) return 2;
  m->addRobotPosition(V3{p[0], p[1], p[2]});
  return 0;
}


int vbo_mesh_generate(void* hv, int use_color, float min_weight, int only_mesh_updated_blocks,
                      int clear_updated_flag) {
  Map* m = static_cast<Map*>(hv);
  const auto t0 = std::chrono::steady_clock::now();
  m->generateMesh(use_color != 0, min_weight, only_mesh_updated_blocks != 0, clear_updated_flag != 0);
  m->last_seconds = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
  return 0;
}
uint64_t vbo_mesh_num_blocks(void* hv) { return static_cast<Map*>(hv)->mesh.size(); }
void vbo_mesh_block_indices(void* hv, int32_t* out) {
  Map* m = static_cast<Map*>(hv);
  std::vector<I3> k;
  for (const auto& kv : m->mesh) k.push_back(kv.first);
  std::sort(k.begin(), k.end(), [](const I3& a, const I3& b) {
    if (a.x != b.x) return a.x < b.x;
    if (a.y != b.y) return a.y < b.y;
    return a.z < b.z;
  });
  for (size_t i = 0; i < k.size(); ++i) {
    out[3 * i] = k[i].x;
    out[3 * i + 1] = k[i].y;
    out[3 * i + 2] = k[i].z;
  }
}
uint64_t vbo_mesh_get(void* hv, const int32_t idx[3], float* vertices, float* normals, uint8_t* colors,
                      int* has_colors, int* updated) {
  Map* m = static_cast<Map*>(hv);
  auto it = m->mesh.find(I3{idx[0], idx[1], idx[2]});
  if (it == m->mesh.end()) return ~0ull;
  const Map::MeshBlk& mb = it->second;
  const size_t n = mb.vertices.size();
  if (vertices && n) std::memcpy(vertices, mb.vertices.data(), n * sizeof(V3));
  if (normals && n) std::memcpy(normals, mb.normals.data(), n * sizeof(V3));
  if (colors && mb.colors.size() == n && n) std::memcpy(colors, mb.colors.data(), n * sizeof(Rgba));
  if (has_colors) *has_colors = (n > 0 && mb.colors.size() == n) ? 1 : 0;
  if (updated) *updated = mb.updated ? 1 : 0;
  return n;
}
int vbo_mc_tables(int32_t*, int32_t*) { return 1; }  // the restatement owns no second copy of the table


}  // extern "C"
namespace {
const uint32_t* g_preset_hashes = nullptr;
struct PresetHash {
  size_t operator()(uint32_t key) const { return static_cast<size_t>(g_preset_hashes[key]); }
};
}  // namespace
extern "C" void vbo_umap_order(const uint32_t* hashes, uint64_t n, uint32_t* out) {
  g_preset_hashes = hashes;
  std::unordered_map<uint32_t, int, PresetHash> m;  // default-constructed like tsdf_integrator.cc:318-322
  for (uint64_t i = 0; i < n; ++i) m[static_cast<uint32_t>(i)] = 0;
  uint64_t p = 0;
  for (const auto& kv : m) out[p++] = kv.first;
}

extern "C" {
}  // extern "C"

// =====================================================================================
// ICP pose refinement (src/alignment/icp.cc, include/voxblox/alignment/icp.h,
// interpolator/interpolator_inl.h -- the nearest-voxel paths icp.cc:126-128 selects).
// Third-party arithmetic (Eigen JacobiSVD / quaternion conversions, minkindr log / exp) is
// restated from the published algorithms; the ICP parity bound is a float tolerance.
// =====================================================================================
namespace {

struct Quat {
  float w, x, y, z;
};
inline Quat qmul(const Quat& a, const Quat& b) {  // Eigen quat_product, scalar path
  return {a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z, a.w * b.x + a.x * b.w + a.y * b.z - a.z * b.y,
          a.w * b.y + a.y * b.w + a.z * b.x - a.x * b.z, a.w * b.z + a.z * b.w + a.x * b.y - a.y * b.x};
}
inline V3 qrot(const Quat& q, V3 p) {  // QuaternionBase::_transformVector
  const V3 qv{q.x, q.y, q.z};
  V3 uv = cross3(qv, p);
  uv = uv + uv;
  return (p + uv * q.w) + cross3(qv, uv);
}
inline Quat qconj(const Quat& q) { return {q.w, -q.x, -q.y, -q.z}; }
struct SE3 {
  Quat q;
  V3 t;
};
inline SE3 se3mul(const SE3& a, const SE3& b) { return {qmul(a.q, b.q), a.t + qrot(a.q, b.t)}; }
inline SE3 se3inv(const SE3& a) {
  const Quat qi = qconj(a.q);
  const V3 r = qrot(qi, a.t);
  return {qi, V3{-r.x, -r.y, -r.z}};
}
// Eigen: quaternion <- rotation matrix (m[r][c])
inline Quat quatFromMatrix(const float m[3][3]) {
  Quat q;
  float t = m[0][0] + m[1][1] + m[2][2];
  if (t > 0.0f) {
    t = std::sqrt(t + 1.0f);
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
    t = std::sqrt(m[i][i] - m[j][j] - m[k][k] + 1.0f);
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
// minkindr RotationQuaternion::log / exp (see oracle/shim/kindr/minimal/quat-transformation.h)
inline V3 quatLog(const Quat& q) {
  const V3 a{q.x, q.y, q.z};
  const float na = norm3(a), eta = q.w;
  float scale;
  if (std::fabs(eta) < na) {
    scale = eta >= 0.0f ? std::acos(eta) / na : -std::acos(-eta) / na;
  } else {
    const float s = std::fabs(na) < std::pow(std::numeric_limits<float>::epsilon(), 0.25f)
                        ? 1.0f + na * na * float(1.0 / 6.0)
                        : std::asin(na) / na;
    scale = eta > 0.0f ? s : -s;
  }
  return a * (2.0f * scale);
}
inline Quat quatExp(V3 d) {
  const double x = d.x, y = d.y, z = d.z;
  const double theta = std::sqrt(x * x + y * y + z * z);
  const double na = theta < std::pow(std::numeric_limits<double>::epsilon(), 0.25) ? 0.5 + (theta * theta) * (1.0 / 48.0)
                                                                                  : std::sin(theta * 0.5) / theta;
  return {static_cast<float>(std::cos(theta * 0.5)), static_cast<float>(x * na), static_cast<float>(y * na),
          static_cast<float>(z * na)};
}

// 3 x 3 proper rotation maximising trace(R H) (= V diag(1, 1, det) U^T of H = U S V^T, icp.h:160-177), by
// the eigen-decomposition of H^T H in double (cyclic Jacobi); returns false on non-finite input.
inline bool rotationFromH3(const float hf[3][3], float r[3][3]) {
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
      for (int j = 0; j < 3; ++j) (i == j ? diag : off) += b[i][j] * b[i][j];
    if (!(off > 1e-60) || off <= 1e-32 * diag) break;
    for (int p = 0; p < 2; ++p)
      for (int q = p + 1; q < 3; ++q) {
        if (b[p][q] == 0.0) continue;
        const double theta = (b[q][q] - b[p][p]) / (2.0 * b[p][q]);
        const double t = (theta >= 0 ? 1.0 : -1.0) / (std::fabs(theta) + std::sqrt(theta * theta + 1.0));
        const double c = 1.0 / std::sqrt(t * t + 1.0), sn = t * c;
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
      if (b[order[j]][order[j]] > b[order[i]][order[i]]) std::swap(order[i], order[j]);
  double u[3][3], vs[3][3], sv[3];
  for (int c = 0; c < 3; ++c) {
    sv[c] = std::sqrt(b[order[c]][order[c]] > 0 ? b[order[c]][order[c]] : 0.0);
    for (int k = 0; k < 3; ++k) vs[k][c] = v[k][order[c]];
  }
  // sqrt of an eigenvalue of H^T H is a relative 1e-16 (s1 / s_c)^2 off: below 1e-4 s1, H v_c / s_c is no
  // longer orthonormal to float accuracy (a planar batch leaves s3 ~ 1e-8 s1 of noise), so complete instead
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
  // completion: H v_c, else the first unit vector left, made orthogonal to the columns before it
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
        for (int i = 0; i < 3; ++i) u[i][c] = w[i] / std::sqrt(nn);
        break;
      }
    }
  float uf[3][3], vf[3][3];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      uf[i][j] = static_cast<float>(u[i][j]);
      vf[i][j] = static_cast<float>(vs[i][j]);
    }
  auto det3 = [](const float m[3][3]) {
    return m[0][0] * (m[1][1] * m[2][2] - m[1][2] * m[2][1]) - m[0][1] * (m[1][0] * m[2][2] - m[1][2] * m[2][0]) +
           m[0][2] * (m[1][0] * m[2][1] - m[1][1] * m[2][0]);
  };
  if (det3(uf) * det3(vf) < 0.0f)
    for (int i = 0; i < 3; ++i) vf[i][2] = vf[i][2] * -1.0f;
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) r[i][j] = vf[i][0] * uf[j][0] + vf[i][1] * uf[j][1] + vf[i][2] * uf[j][2];
  return true;
}

// minkindr's Rotation::isValidRotationMatrix with the threshold of oracle/shim/kindr (1000 float epsilons)
inline bool isValidRotation(const float m[3][3]) {
  const float thr = 1000.0f * std::numeric_limits<float>::epsilon();
  const float det = m[0][0] * (m[1][1] * m[2][2] - m[1][2] * m[2][1]) - m[0][1] * (m[1][0] * m[2][2] - m[1][2] * m[2][0]) +
                    m[0][2] * (m[1][0] * m[2][1] - m[1][1] * m[2][0]);
  if (std::fabs(det - 1.0f) > thr) return false;
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j)
      if (std::fabs(m[i][0] * m[j][0] + m[i][1] * m[j][1] + m[i][2] * m[j][2] - (i == j ? 1.0f : 0.0f)) > thr) return false;
  return true;
}

struct IcpStep {
  bool ok = false;
  SE3 delta{};
  float info[6] = {0, 0, 0, 0, 0, 0};
};

struct IcpRunner {
  const Map& m;
  vbo_icp_config cfg;
  float block_size_inv;

  IcpRunner(const Map& map, const vbo_icp_config& c) : m(map), cfg(c) {
    block_size_inv = static_cast<float>(1.0 / m.block_size);  // Layer ctor, core/layer.h:41
  }

  // Interpolator::getNearestDistance (interpolator_inl.h:330-345): Layer::getBlockPtrByCoordinates,
  // Block::getVoxelByCoordinates (truncated voxel index, block_inl.h:30-40), observed = weight > 1e-6
  bool nearestDistance(V3 p, float* d, bool* has_block) const {
    const L3 bi = gridIndex(p, block_size_inv);
    auto it = m.tsdf.find(I3{static_cast<int>(bi.x), static_cast<int>(bi.y), static_cast<int>(bi.z)});
    if (it == m.tsdf.end()) {
      *has_block = false;
      return false;
    }
    *has_block = true;
    const V3 origin{static_cast<float>(static_cast<int>(bi.x)) * m.block_size, static_cast<float>(static_cast<int>(bi.y)) * m.block_size,
                    static_cast<float>(static_cast<int>(bi.z)) * m.block_size};
    const L3 vi = gridIndex(p - origin, m.voxel_size_inv);
    const int mx = m.vps - 1;
    const int x = std::max(std::min(static_cast<int>(vi.x), mx), 0), y = std::max(std::min(static_cast<int>(vi.y), mx), 0),
              z = std::max(std::min(static_cast<int>(vi.z), mx), 0);
    const TsdfVox& v = it->second->vox[static_cast<size_t>(x + m.vps * (y + m.vps * z))];
    *d = v.distance;
    return static_cast<double>(v.weight) > 1e-6;
  }
  // Interpolator::getGradient, interpolate = false (interpolator_inl.h:48-77)
  bool gradient(V3 p, V3* g) const {
    float d;
    bool has_block;
    nearestDistance(p, &d, &has_block);
    if (!has_block) return false;
    float gr[3] = {0.0f, 0.0f, 0.0f};
    for (int i = 0; i < 3; ++i)
      for (int sign = -1; sign <= 1; sign += 2) {
        V3 q = p;
        const float off = static_cast<float>(sign) * m.voxel_size;
        (i == 0 ? q.x : i == 1 ? q.y : q.z) += off;
        float od;
        bool hb;
        if (!nearestDistance(q, &od, &hb)) return false;
        gr[i] = gr[i] + od * static_cast<float>(sign);
      }
    const float den = 2 * m.voxel_size;
    *g = V3{gr[0] / den, gr[1] / den, gr[2] / den};
    return true;
  }

  // ICP::stepICP = matchPoints + getTransformFromMatchedPoints (icp.cc:104-169, :50-80, icp.h:146-187)
  IcpStep step(const std::vector<V3>& pts, size_t start, const SE3& T) const {
    IcpStep out;
    const size_t mb = static_cast<size_t>(cfg.mini_batch_size);
    std::vector<V3> src, tgt;
    float info[6];
    for (float& v : info) v = kEps;
    const Pose pose{T.q.w, T.q.x, T.q.y, T.q.z, T.t};
    for (size_t i = start; i < std::min(pts.size(), start + mb); ++i) {
      const V3 p = pose.apply(pts[i]);
      const L3 vidx = gridIndex(p, m.voxel_size_inv);
      float dist;
      bool hb;
      V3 g;
      if (nearestDistance(p, &dist, &hb) && gradient(p, &g) && sqnorm3(g) > 0.1f) {
        g = unit3(g);
        const V3 q = p - T.t;  // addNormalizedPointInfo (icp.cc:82-102)
        info[0] = info[0] + 2.0f * (g.x * g.x);
        info[1] = info[1] + 2.0f * (g.y * g.y);
        info[2] = info[2] + 2.0f * (g.z * g.z);
        info[3] = info[3] + 2.0f * (q.y * q.y * g.z * g.z + q.z * q.z * g.y * g.y);
        info[4] = info[4] + 2.0f * (q.x * q.x * g.z * g.z + q.z * q.z * g.x * g.x);
        info[5] = info[5] + 2.0f * (q.x * q.x * g.y * g.y + q.y * q.y * g.x * g.x);
        const V3 centre = centerPoint(vidx, m.voxel_size);
        dist = dist + dot3(g, p - centre);
        src.push_back(p);
        tgt.push_back(p - g * dist);
      }
    }
    for (int k = 0; k < 6; ++k) out.info[k] = info[k];
    const int n = static_cast<int>(src.size());
    if (n < std::max(3, static_cast<int>(cfg.mini_batch_size * cfg.min_match_ratio))) return out;
    V3 sc = src[0], tc = tgt[0];
    for (int i = 1; i < n; ++i) {
      sc = sc + src[i];
      tc = tc + tgt[i];
    }
    sc = sc / static_cast<float>(n);
    tc = tc / static_cast<float>(n);
    const int dim = cfg.refine_roll_pitch ? 3 : 2;
    float h[3][3] = {{0, 0, 0}, {0, 0, 0}, {0, 0, 0}};
    for (int k = 0; k < n; ++k) {
      const V3 s = src[k] - sc, t = tgt[k] - tc;
      const float sv[3] = {s.x, s.y, s.z}, tv[3] = {t.x, t.y, t.z};
      for (int i = 0; i < dim; ++i)
        for (int j = 0; j < dim; ++j) h[i][j] = h[i][j] + sv[i] * tv[j];
    }
    float r[3][3] = {{1, 0, 0}, {0, 1, 0}, {0, 0, 1}};
    if (dim == 2) {
      // the proper rotation V diag(1, det) U^T of the 2 x 2 SVD maximises trace(R H): closed form
      const float a = h[0][0] + h[1][1], b = h[0][1] - h[1][0];
      const float nrm = std::sqrt(a * a + b * b);
      const float c = nrm == 0.0f ? 1.0f : a / nrm, s = nrm == 0.0f ? 0.0f : b / nrm;  // H = 0: SVD U = V = I
      r[0][0] = c;
      r[0][1] = -s;
      r[1][0] = s;
      r[1][1] = c;
    } else if (!rotationFromH3(h, r)) {
      return out;
    }
    float sum = 0;
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) sum += r[i][j];
    if (!std::isfinite(sum) || !isValidRotation(r)) return out;  // icp.h:183-189
    out.delta.q = quatFromMatrix(r);
    out.delta.t = tc - qrot(out.delta.q, sc);
    out.ok = true;
    return out;
  }
};

}  // namespace

extern "C" void vbo_icp_shuffle(uint64_t n, uint32_t seed, uint32_t* out) {
  std::iota(out, out + n, 0u);
  std::shuffle(out, out + n, std::default_random_engine(seed));  // the C++ library's own, as icp.cc:231-233 calls it
}

extern "C" int vbo_icp_run(void* hv, const vbo_icp_config* c, const float* xyz, uint64_t n, const float q[4],
                           const float t[3], uint32_t seed, float out_q[4], float out_t[3], uint64_t* num_updates) {
  Map& m = *static_cast<Map*>(hv);
  if (c->num_threads < 1 || c->mini_batch_size < 1) return 2;
  const auto t0 = std::chrono::steady_clock::now();
  std::vector<uint32_t> perm(n);
  vbo_icp_shuffle(n, seed, perm.data());
  std::vector<V3> pts(n);
  for (uint64_t i = 0; i < n; ++i) pts[i] = V3{xyz[3 * perm[i]], xyz[3 * perm[i] + 1], xyz[3 * perm[i] + 2]};
  IcpRunner run(m, *c);
  SE3 cur{Quat{q[0], q[1], q[2], q[3]}, V3{t[0], t[1], t[2]}};
  float base[6] = {c->inital_translation_weighting, c->inital_translation_weighting, c->inital_translation_weighting,
                   c->inital_rotation_weighting,    c->inital_rotation_weighting,    c->inital_rotation_weighting};
  const int T = c->num_threads;
  std::vector<SE3> snapshot(T, cur);  // runThread's current_thread_T_tsdf_sensor (icp.cc:178-182)
  std::vector<char> alive(T, 1);
  size_t next_idx = 0, updates = 0;
  const size_t mb = static_cast<size_t>(c->mini_batch_size);
  for (;;) {
    // one round of the round-robin schedule: fetch_add in thread order, match, fuse in thread order
    std::vector<std::pair<int, size_t>> jobs;
    for (int w = 0; w < T; ++w) {
      if (!alive[w]) continue;
      const size_t start = next_idx;
      next_idx += mb;
      if (static_cast<float>(start) > c->subsample_keep_ratio * static_cast<float>(n)) {  // icp.cc:186-188
        alive[w] = 0;
        continue;
      }
      jobs.emplace_back(w, start);
    }
    if (jobs.empty()) break;
    std::vector<IcpStep> res(jobs.size());
    for (size_t k = 0; k < jobs.size(); ++k) res[k] = run.step(pts, jobs[k].second, snapshot[jobs[k].first]);
    for (size_t k = 0; k < jobs.size(); ++k) {
      if (!res[k].ok) continue;
      // icp.cc:195-213
      const SE3 t_temp = se3mul(res[k].delta, cur);
      SE3 d = se3mul(se3inv(cur), t_temp);
      const V3 w3 = quatLog(d.q);
      const float lg[6] = {d.t.x, d.t.y, d.t.z, w3.x, w3.y, w3.z};
      float wl[6];
      for (int i = 0; i < 6; ++i) {
        const float weight = res[k].info[i] / (base[i] + res[k].info[i]);
        wl[i] = weight * lg[i];
      }
      d = SE3{quatExp(V3{wl[3], wl[4], wl[5]}), V3{wl[0], wl[1], wl[2]}};
      for (int i = 0; i < 6; ++i) base[i] = base[i] + res[k].info[i];
      cur = se3mul(cur, d);
      snapshot[jobs[k].first] = cur;
      ++updates;
    }
  }
  out_q[0] = cur.q.w;
  out_q[1] = cur.q.x;
  out_q[2] = cur.q.y;
  out_q[3] = cur.q.z;
  out_t[0] = cur.t.x;
  out_t[1] = cur.t.y;
  out_t[2] = cur.t.z;
  if (num_updates) *num_updates = updates;
  m.last_seconds = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
  return 0;
}

