// Layer files (.vxblx): Layer::saveToFile / io::LoadBlocksFromFile
// (voxblox/include/voxblox/core/layer_inl.h:81-189, io/layer_io_inl.h:13-129,
// src/utils/protobuf_utils.cc:9-98) straight from / into the device map.  SURVEY.md 8(f) N2.
//
// File = varint32(number of messages) | varint32(size) LayerProto | { varint32(size) BlockProto }
// (proto/voxblox/Layer.proto, Block.proto, proto2).  The reference links libprotobuf; the two
// messages are six scalar fields and one repeated uint32, so the wire format is written and parsed
// here directly: fields in ascending number, every field Block::getProto / Layer::getProto sets is
// present (proto2 writes set fields even when zero), `repeated uint32 voxel_data = 7` unpacked
// (proto2 default: one tag byte 0x38 + varint per word); the parser also accepts the packed form.
// The voxel words themselves are packed on the device (vbx_blocks.cu, k_serialize_blocks).
#include <cmath>
#include <cstdio>
#include <cstring>
#include <limits>
#include <string>
#include <vector>

#include "vbx_engine.h"

namespace vbx {

int upload_blocks(vbx_ctx* c, int layer, const int32_t* idx3, uint64_t m, const void* voxels,
                  const uint8_t* updated_bits, int serialized);

namespace {

inline void put_varint(std::string* o, uint64_t v) {
  while (v >= 0x80u) {
    o->push_back((char)((v & 0x7fu) | 0x80u));
    v >>= 7;
  }
  o->push_back((char)v);
}
inline void put_double(std::string* o, int field, double v) {
  put_varint(o, ((uint64_t)field << 3) | 1u);
  char b[8];
  std::memcpy(b, &v, 8);
  o->append(b, 8);
}

struct Reader {
  const uint8_t* p;
  const uint8_t* end;
  bool ok = true;
  uint64_t varint() {
    uint64_t v = 0;
    for (int shift = 0; shift < 64; shift += 7) {
      if (p >= end) {
        ok = false;
        return 0;
      }
      const uint8_t b = *p++;
      v |= (uint64_t)(b & 0x7fu) << shift;
      if (!(b & 0x80u)) return v;
    }
    ok = false;
    return 0;
  }
  double f64() {
    if (end - p < 8) {
      ok = false;
      return 0;
    }
    double v;
    std::memcpy(&v, p, 8);
    p += 8;
    return v;
  }
  void skip(uint32_t wire_type) {
    if (wire_type == 0) {
      varint();
    } else if (wire_type == 1) {
      if (end - p < 8) ok = false; else p += 8;
    } else if (wire_type == 5) {
      if (end - p < 4) ok = false; else p += 4;
    } else if (wire_type == 2) {
      const uint64_t n = varint();
      if (!ok || (uint64_t)(end - p) < n) ok = false; else p += n;
    } else {
      ok = false;
    }
  }
};

}  // namespace

// Layer::getProto, core/layer_inl.h:41-51
std::string encode_layer_proto(double voxel_size, uint32_t vps, const char* type) {
  std::string o;
  put_double(&o, 1, voxel_size);
  put_varint(&o, (2u << 3) | 0u);
  put_varint(&o, vps);
  const size_t n = std::strlen(type);
  put_varint(&o, (3u << 3) | 2u);
  put_varint(&o, n);
  o.append(type, n);
  return o;
}

// Block::getProto, core/block_inl.h:91-109
void encode_block_proto(std::string* o, int32_t vps, double voxel_size, const double origin[3], bool has_data,
                        const uint32_t* words, size_t n_words) {
  o->clear();
  o->reserve(64 + 6 * n_words);
  put_varint(o, (1u << 3) | 0u);
  put_varint(o, (uint64_t)(int64_t)vps);  // int32: sign-extended to 64 bits on the wire
  put_double(o, 2, voxel_size);
  put_double(o, 3, origin[0]);
  put_double(o, 4, origin[1]);
  put_double(o, 5, origin[2]);
  put_varint(o, (6u << 3) | 0u);
  o->push_back(has_data ? 1 : 0);
  for (size_t i = 0; i < n_words; ++i) {
    o->push_back((char)0x38);  // field 7, varint
    put_varint(o, words[i]);
  }
}

struct BlockMsg {
  int32_t vps = 0;
  double voxel_size = 0, origin[3] = {0, 0, 0};
  bool has_data = false;
  std::vector<uint32_t> words;
};

bool decode_block_proto(const uint8_t* msg, size_t len, BlockMsg* b) {
  Reader r{msg, msg + len};
  b->words.clear();
  while (r.ok && r.p < r.end) {
    const uint64_t tag = r.varint();
    const uint32_t field = (uint32_t)(tag >> 3), wt = (uint32_t)(tag & 7u);
    if (field == 1 && wt == 0) {
      b->vps = (int32_t)r.varint();
    } else if (field == 2 && wt == 1) {
      b->voxel_size = r.f64();
    } else if (field >= 3 && field <= 5 && wt == 1) {
      b->origin[field - 3] = r.f64();
    } else if (field == 6 && wt == 0) {
      b->has_data = r.varint() != 0;
    } else if (field == 7 && wt == 0) {
      b->words.push_back((uint32_t)r.varint());
    } else if (field == 7 && wt == 2) {  // packed encoding of the same field
      const uint64_t n = r.varint();
      if (!r.ok || (uint64_t)(r.end - r.p) < n) return false;
      Reader q{r.p, r.p + n};
      while (q.ok && q.p < q.end) b->words.push_back((uint32_t)q.varint());
      if (!q.ok) return false;
      r.p += n;
    } else {
      r.skip(wt);
    }
  }
  return r.ok;
}

struct LayerMsg {
  double voxel_size = 0;
  uint32_t vps = 0;
  std::string type;
};

bool decode_layer_proto(const uint8_t* msg, size_t len, LayerMsg* l) {
  Reader r{msg, msg + len};
  while (r.ok && r.p < r.end) {
    const uint64_t tag = r.varint();
    const uint32_t field = (uint32_t)(tag >> 3), wt = (uint32_t)(tag & 7u);
    if (field == 1 && wt == 1) {
      l->voxel_size = r.f64();
    } else if (field == 2 && wt == 0) {
      l->vps = (uint32_t)r.varint();
    } else if (field == 3 && wt == 2) {
      const uint64_t n = r.varint();
      if (!r.ok || (uint64_t)(r.end - r.p) < n) return false;
      l->type.assign(reinterpret_cast<const char*>(r.p), n);
      r.p += n;
    } else {
      r.skip(wt);
    }
  }
  return r.ok;
}

static const char* layer_type(int layer) { return layer == VBX_LAYER_TSDF ? "tsdf" : "esdf"; }  // core/voxel.h:52-53

// Layer::saveToFile(file_path, clear_file), core/layer_inl.h:81-157
int save_layer(vbx_ctx* c, int layer, const char* path, int clear_file) {
  if (layer == VBX_LAYER_ESDF && !c->esdf.ready) return fail(c, VBX_E_STATE, "no ESDF layer");
  const size_t wpv = layer == VBX_LAYER_TSDF ? 3 : 2;
  const size_t wpb = wpv * c->vox_per_block;
  uint64_t n = 0;
  std::vector<int32_t> idx(3 * (size_t)std::max<uint32_t>(c->n_blocks, 1));
  std::vector<uint32_t> words((size_t)std::max<uint32_t>(c->n_blocks, 1) * wpb);
  if (c->n_blocks) {
    if (int rc = mirror_updated(c, layer, 0, 0, idx.data(), words.data(), nullptr, c->n_blocks, &n, 1)) return rc;
  }
  FILE* f = std::fopen(path, clear_file ? "wb" : "ab");
  if (!f) return fail(c, VBX_E_INVALID, std::string("Could not open file for writing: ") + path);
  std::string out;
  put_varint(&out, 1u + n);  // one layer header and then all the blocks, cc:128-131
  const std::string header = encode_layer_proto((double)c->voxel_size, (uint32_t)(1u << c->L), layer_type(layer));
  put_varint(&out, header.size());
  out += header;
  bool ok = std::fwrite(out.data(), 1, out.size(), f) == out.size();
  const float block_size = c->voxel_size * (float)(1u << c->L);  // Layer ctor, core/layer.h:44-50
  std::string msg;
  for (uint64_t b = 0; ok && b < n; ++b) {
    // Block origin = getOriginPointFromGridIndex(index, block_size) in float (core/common.h:196-201)
    const double origin[3] = {(double)((float)idx[3 * b] * block_size), (double)((float)idx[3 * b + 1] * block_size),
                              (double)((float)idx[3 * b + 2] * block_size)};
    // has_data_: false for every block the integrators made (SURVEY a18); true only where a loaded file said so
    const bool has_data = c->has_data_keys[layer == VBX_LAYER_ESDF ? 1 : 0].count(pack3(idx[3 * b], idx[3 * b + 1], idx[3 * b + 2])) != 0;
    encode_block_proto(&msg, (int32_t)(1u << c->L), (double)c->voxel_size, origin, has_data, words.data() + b * wpb, wpb);
    out.clear();
    put_varint(&out, msg.size());
    ok = std::fwrite(out.data(), 1, out.size(), f) == out.size() && std::fwrite(msg.data(), 1, msg.size(), f) == msg.size();
  }
  ok = (std::fclose(f) == 0) && ok;
  if (!ok) return fail(c, VBX_E_INVALID, std::string("write error: ") + path);
  return VBX_OK;
}

// io::LoadBlocksFromFile(file_path, kReplace, multiple_layer_support = true, layer), io/layer_io_inl.h:13-90
int load_layer(vbx_ctx* c, int layer, const char* path, uint64_t* n_loaded) {
  *n_loaded = 0;
  if (layer == VBX_LAYER_ESDF && !c->esdf.ready) return fail(c, VBX_E_STATE, "no ESDF layer");
  FILE* f = std::fopen(path, "rb");
  if (!f) return fail(c, VBX_E_NOT_FOUND, std::string("Could not open protobuf file to load layer: ") + path);
  std::vector<uint8_t> data;
  {
    std::fseek(f, 0, SEEK_END);
    const long sz = std::ftell(f);
    std::fseek(f, 0, SEEK_SET);
    data.resize(sz > 0 ? (size_t)sz : 0);
    const size_t got = data.empty() ? 0 : std::fread(data.data(), 1, data.size(), f);
    std::fclose(f);
    if (got != data.size()) return fail(c, VBX_E_INVALID, std::string("read error: ") + path);
  }
  Reader r{data.data(), data.data() + data.size()};
  const size_t wpv = layer == VBX_LAYER_TSDF ? 3 : 2;
  const size_t wpb = wpv * c->vox_per_block;
  const float block_size = c->voxel_size * (float)(1u << c->L);
  const float block_size_inv = (float)(1.0 / (double)block_size);
  bool layer_found = false;
  while (!layer_found && r.p < r.end) {
    const uint64_t num_protos = r.varint();
    if (!r.ok) return fail(c, VBX_E_INVALID, "Could not read number of messages.");
    if (num_protos == 0) return fail(c, VBX_E_INVALID, "Empty protobuf file!");
    const uint64_t hsize = r.varint();
    if (!r.ok || hsize == 0 || (uint64_t)(r.end - r.p) < hsize) return fail(c, VBX_E_INVALID, "Could not read layer protobuf message.");
    LayerMsg lm;
    if (!decode_layer_proto(r.p, hsize, &lm)) return fail(c, VBX_E_INVALID, "Could not parse layer protobuf message.");
    r.p += hsize;
    // Layer::isCompatible(LayerProto), core/layer_inl.h:237-260
    const bool compatible = std::fabs(lm.voxel_size - (double)c->voxel_size) < (double)std::numeric_limits<float>::epsilon() &&
                            lm.vps == (1u << c->L) && lm.type == layer_type(layer);
    std::vector<int32_t> idx;
    std::vector<uint32_t> words;
    std::vector<uint8_t> has_data;
    BlockMsg bm;
    for (uint64_t b = 0; b + 1 < num_protos; ++b) {
      const uint64_t bsize = r.varint();
      if (!r.ok || bsize == 0 || (uint64_t)(r.end - r.p) < bsize) {
        return fail(c, VBX_E_INVALID, "Could not read block protobuf message number " + std::to_string(b));
      }
      if (compatible) {
        if (!decode_block_proto(r.p, bsize, &bm)) return fail(c, VBX_E_INVALID, "Could not parse block protobuf message.");
        // Layer::isCompatible(BlockProto) + Block(BlockProto)'s CHECK_EQ on the word count
        if (!(std::fabs(bm.voxel_size - (double)c->voxel_size) < (double)std::numeric_limits<float>::epsilon()) ||
            bm.vps != (int32_t)(1u << c->L) || bm.words.size() != wpb) {
          return fail(c, VBX_E_INVALID, "The blocks from this protobuf are not compatible with this layer!");
        }
        // getGridIndexFromOriginPoint<BlockIndex>(origin, block_size_inv), core/common.h:171-177
        for (int a = 0; a < 3; ++a) idx.push_back((int32_t)std::round((float)bm.origin[a] * block_size_inv));
        words.insert(words.end(), bm.words.begin(), bm.words.end());
        has_data.push_back(bm.has_data ? 1 : 0);
      }
      r.p += bsize;
    }
    if (compatible) {
      layer_found = true;
      uint64_t m = idx.size() / 3;
      // kReplace: a block listed twice keeps the LAST payload, like block_map_[index] = block
      // (io/layer_io_inl.h:71-73).  One upload scatters all blocks concurrently, so earlier duplicates are
      // dropped here, on the host.
      {
        std::unordered_map<uint64_t, uint64_t> last;
        for (uint64_t b = 0; b < m; ++b) last[pack3(idx[3 * b], idx[3 * b + 1], idx[3 * b + 2])] = b;
        if (last.size() != m) {
          uint64_t w = 0;
          for (uint64_t b = 0; b < m; ++b) {
            if (last[pack3(idx[3 * b], idx[3 * b + 1], idx[3 * b + 2])] != b) continue;
            if (w != b) {
              std::copy(idx.begin() + 3 * b, idx.begin() + 3 * b + 3, idx.begin() + 3 * w);
              std::copy(words.begin() + b * wpb, words.begin() + (b + 1) * wpb, words.begin() + w * wpb);
              has_data[w] = has_data[b];
            }
            ++w;
          }
          m = w;
        }
      }
      std::vector<uint8_t> upd(m, (uint8_t)7);  // updated().set(), core/layer_inl.h:227
      if (m) {
        if (int rc = upload_blocks(c, layer, idx.data(), m, words.data(), upd.data(), 1)) return rc;
      }
      std::unordered_set<uint64_t>& hd = c->has_data_keys[layer == VBX_LAYER_ESDF ? 1 : 0];
      for (uint64_t b = 0; b < m; ++b) {
        const uint64_t key = pack3(idx[3 * b], idx[3 * b + 1], idx[3 * b + 2]);
        if (has_data[b]) {
          hd.insert(key);
        } else {
          hd.erase(key);
        }
      }
      *n_loaded = m;
    }
  }
  if (!layer_found) return fail(c, VBX_E_NOT_FOUND, "The layer information read from file is not compatible with the current layer!");
  return VBX_OK;
}

}  // namespace vbx

using namespace vbx;

extern "C" {

// host-only helpers: the exact bytes libprotobuf produces for Layer::getProto / Block::getProto
// (checked against a real protobuf implementation in tests/test_proto_io.py, no GPU needed)
int vbx_proto_encode_layer(double voxel_size, uint32_t voxels_per_side, const char* type, uint8_t* out, uint64_t cap,
                           uint64_t* n) {
  if (!type || !n) return VBX_E_INVALID;
  const std::string s = encode_layer_proto(voxel_size, voxels_per_side, type);
  *n = s.size();
  if (out && cap >= s.size()) std::memcpy(out, s.data(), s.size());
  return VBX_OK;
}

int vbx_proto_encode_block(int32_t voxels_per_side, double voxel_size, const double origin[3], int has_data,
                           const uint32_t* words, uint64_t n_words, uint8_t* out, uint64_t cap, uint64_t* n) {
  if (!origin || !n || (n_words && !words)) return VBX_E_INVALID;
  std::string s;
  encode_block_proto(&s, voxels_per_side, voxel_size, origin, has_data != 0, words, n_words);
  *n = s.size();
  if (out && cap >= s.size()) std::memcpy(out, s.data(), s.size());
  return VBX_OK;
}

int vbx_proto_decode_block(const uint8_t* msg, uint64_t len, int32_t* voxels_per_side, double* voxel_size,
                           double origin[3], int* has_data, uint32_t* words, uint64_t cap_words, uint64_t* n_words) {
  if (!msg || !n_words) return VBX_E_INVALID;
  BlockMsg b;
  if (!decode_block_proto(msg, len, &b)) return VBX_E_INVALID;
  if (voxels_per_side) *voxels_per_side = b.vps;
  if (voxel_size) *voxel_size = b.voxel_size;
  if (origin) std::memcpy(origin, b.origin, sizeof(b.origin));
  if (has_data) *has_data = b.has_data ? 1 : 0;
  *n_words = b.words.size();
  if (words && cap_words >= b.words.size()) std::memcpy(words, b.words.data(), b.words.size() * sizeof(uint32_t));
  return VBX_OK;
}

int vbx_save_layer(vbx_ctx* c, int layer, const char* path, int clear_file) {
  if (!c || !path || !*path) return fail(c, VBX_E_INVALID, "null argument");  // CHECK(!file_path.empty())
  if (cudaSetDevice(c->device) != cudaSuccess) return fail(c, VBX_E_CUDA, "cudaSetDevice");
  if (int rc = drain_async(c)) return rc;
  return save_layer(c, layer, path, clear_file);
}

int vbx_load_layer(vbx_ctx* c, int layer, const char* path, uint64_t* n_loaded) {
  if (!c || !path || !*path || !n_loaded) return fail(c, VBX_E_INVALID, "null argument");
  if (cudaSetDevice(c->device) != cudaSuccess) return fail(c, VBX_E_CUDA, "cudaSetDevice");
  if (int rc = drain_async(c)) return rc;
  return load_layer(c, layer, path, n_loaded);
}

}  // extern "C"
