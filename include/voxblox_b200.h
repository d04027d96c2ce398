/* voxblox_b200 -- C-ABI of the H100-native TSDF / ESDF integration engine.
 *
 * This is the drop-in boundary for the ONE hot path of ethz-asl/voxblox that this
 * repository accelerates (SURVEY.md section 8b).  The reference has no FFI today;
 * its "operator API" is the C++ virtual
 *     TsdfIntegratorBase::integratePointCloud(T_G_C, points_C, colors, freespace)
 *         voxblox/include/voxblox/integrator/tsdf_integrator.h:100-103
 * and
 *     EsdfIntegrator::updateFromTsdfLayer(clear_updated_flag) / ...Batch()
 *         voxblox/include/voxblox/integrator/esdf_integrator.h:101-106
 * operating on Layer<TsdfVoxel> / Layer<EsdfVoxel> (core/layer.h:24-296).
 * Each entry point below names the reference interface it replaces; the voxblox-
 * side adapter that binds them (a TsdfIntegratorBase subclass registered in
 * TsdfIntegratorFactory::create) is include/voxblox_b200/gpu_integrators.h and is
 * described in INTEGRATION.md.
 *
 * Conventions: plain pointers and sizes only; every function returns 0 on success
 * or a VBX_E_* code, with a message retrievable through vbx_last_error() (the
 * reference aborts through glog CHECK/LOG(FATAL); the adapter maps non-zero to
 * LOG(FATAL) to keep that behaviour).  A context is NOT thread safe, exactly like
 * integratePointCloud (tsdf_integrator.h:95); calls are synchronous at return
 * unless stated otherwise.  Voxel payloads use the reference's in-memory structs:
 *   TsdfVoxel 12 B = f32 distance, f32 weight, u8 r,g,b,a        (core/voxel.h:12-16)
 *   EsdfVoxel 20 B = f32 distance, u8 observed, hallucinated,
 *                    in_queue, fixed, i32 parent[3]               (core/voxel.h:18-37)
 * in linear order x + vps*(y + vps*z) (core/block_inl.h:12-27).
 */
#ifndef VOXBLOX_B200_H_
#define VOXBLOX_B200_H_

#include <stddef.h>
#include <stdint.h>

#if defined(__GNUC__)
#define VBX_API __attribute__((visibility("default")))
#else
#define VBX_API
#endif

#ifdef __cplusplus
extern "C" {
#endif

#define VBX_OK 0
#define VBX_E_INVALID 1      /* bad argument / unknown integrator type (cc:11,22,41) */
#define VBX_E_CUDA 2         /* CUDA runtime error                                    */
#define VBX_E_CAPACITY 3     /* block pool / scratch capacity exceeded                */
#define VBX_E_NOT_FOUND 4    /* block does not exist                                  */
#define VBX_E_STATE 5        /* call order (e.g. ESDF update before vbx_esdf_create)  */

/* TsdfIntegratorType, tsdf_integrator.h:30-41 */
#define VBX_SIMPLE 1
#define VBX_MERGED 2
#define VBX_FAST 3

#define VBX_LAYER_TSDF 0
#define VBX_LAYER_ESDF 1

/* Update::Status bits of Block::updated(), core/block.h:15-18 */
#define VBX_UPDATED_MAP 1
#define VBX_UPDATED_MESH 2
#define VBX_UPDATED_ESDF 4
/* Not a voxblox bit: the engine's own "changed since it was last mirrored" mark, set by every TSDF / ESDF
 * update of a block next to Block::updated().  Accepted in the updated_mask / clear_mask of
 * vbx_mirror_updated and vbx_serialize_updated (never reported back), so that an incremental host mirror
 * does not depend on -- or disturb -- the three bits above, which belong to their consumers. */
#define VBX_UPDATED_MIRROR 8

typedef struct vbx_ctx vbx_ctx;

/* POD mirror of TsdfIntegratorBase::Config, tsdf_integrator.h:56-89 (defaults there).
 * integration_order_mode: 0 = "mixed", 1 = "sorted" (integrator_utils.cc:5-15).
 * integrator_threads is accepted for API parity and ignored: the device applies
 * every voxel's updates in one fixed order (DESIGN.md, "update order").
 * Fast only: max_integration_time_s <= 0 or NaN integrates no point of a call, as in the reference;
 * a positive limit is wall-clock time and is not enforced.  clear_checks_every_n_frames counts the
 * Fast calls of this context; the reference's counter is one static shared by every Fast integrator
 * of the process (tsdf_integrator.cc:564). */
typedef struct vbx_tsdf_config {
  float default_truncation_distance;
  float max_weight;
  int32_t voxel_carving_enabled;
  float min_ray_length_m;
  float max_ray_length_m;
  int32_t use_const_weight;
  int32_t allow_clear;
  int32_t use_weight_dropoff;
  int32_t use_sparsity_compensation_factor;
  float sparsity_compensation_factor;
  int32_t integrator_threads;
  int32_t integration_order_mode;
  int32_t enable_anti_grazing;
  float start_voxel_subsampling_factor;
  int32_t max_consecutive_ray_collisions;
  int32_t clear_checks_every_n_frames;
  float max_integration_time_s;
} vbx_tsdf_config;

/* POD mirror of EsdfIntegrator::Config, esdf_integrator.h:29-78. */
typedef struct vbx_esdf_config {
  int32_t full_euclidean_distance;
  float max_distance_m;
  float min_distance_m;
  float default_distance_m;
  float min_diff_m;
  float min_weight;
  int32_t num_buckets;
  int32_t multi_queue;
  int32_t add_occupied_crust;
  float clear_sphere_radius;
  float occupied_sphere_radius;
} vbx_esdf_config;

/* Engine sizing (no reference counterpart: the CPU map grows with make_shared).
 * Zero in any field selects the default in brackets. */
typedef struct vbx_engine_options {
  int32_t device;                 /* CUDA device ordinal [current]                    */
  uint32_t max_blocks;            /* voxel-block pool capacity [32768 = 1.5 GiB TSDF] */
  uint32_t max_points_per_scan;   /* [1 << 20]                                        */
  uint64_t max_updates_per_pass;  /* ray-voxel update records per pass [1 << 26]      */
  int32_t rank;                   /* this process' rank in the group [0]              */
  int32_t world_size;             /* block-ownership shards of ONE map [1], see below */
} vbx_engine_options;

/* Layer<TsdfVoxel>(voxel_size, voxels_per_side) + TsdfIntegratorBase(config, layer)
 * (core/layer.h:36-47, tsdf_integrator.cc:53-80). voxels_per_side must be a power
 * of two <= 16 (the reference CHECKs the power of two, core/common.h:239). */
VBX_API int vbx_create(const vbx_tsdf_config* cfg, float voxel_size, int voxels_per_side,
               const vbx_engine_options* opt, vbx_ctx** out);
VBX_API void vbx_destroy(vbx_ctx* ctx);
VBX_API const char* vbx_last_error(const vbx_ctx* ctx);
VBX_API const char* vbx_version(void);

/* TsdfIntegratorBase::getConfig (tsdf_integrator.h:106) */
VBX_API int vbx_get_tsdf_config(const vbx_ctx* ctx, vbx_tsdf_config* out);

/* {Simple,Merged,Fast}TsdfIntegrator::integratePointCloud
 * (tsdf_integrator.cc:242-267, 307-338, 555-590).  kind = VBX_SIMPLE|MERGED|FAST,
 * T_G_C = (q_wxyz, t), xyz = 3n floats points_C, rgba = 4n bytes, HOST memory.
 * Copies the cloud to the device, integrates, and returns after the stream has
 * drained (the reference's call is synchronous too). */
VBX_API int vbx_tsdf_integrate(vbx_ctx* ctx, int kind, const float q_wxyz[4], const float t[3],
                       const float* xyz, const uint8_t* rgba, uint64_t n, int freespace);
/* Asynchronous submission (no reference counterpart: its call is synchronous).  Enqueues the scan
 * and returns.  A scan passes through four stages on separate streams (front: transform, bundle
 * sort, bundle fold -- walk: ray walk with block creation -- sort: update-record sort -- apply),
 * so the stages of up to six consecutive scans overlap; stages that touch the map run strictly in
 * submission order, and the result equals the synchronous calls' bit for bit.  Host buffers
 * (inputs_on_device = 0) should be page-locked and must then stay untouched until the scan
 * completed (vbx_sync, or six submissions later); pageable buffers are staged before the call
 * returns and may be reused at once.  Counters and errors of a scan surface at the next
 * synchronous call / vbx_sync (a failed scan is reported, not retried: a clearing point beyond
 * the compact key range -- 511 voxels -- drops that scan and switches later ones to wide keys).
 * Configurations whose front half touches the map (Fast, anti-grazing, "sorted" order) fall back
 * to the synchronous path.  The extra buffers are allocated on the first call. */
VBX_API int vbx_tsdf_integrate_async(vbx_ctx* ctx, int kind, const float q_wxyz[4], const float t[3],
                             const float* xyz, const uint8_t* rgba, uint64_t n, int freespace,
                             int inputs_on_device);
/* Same, with xyz / rgba already resident in DEVICE memory (no copies). */
VBX_API int vbx_tsdf_integrate_device(vbx_ctx* ctx, int kind, const float q_wxyz[4], const float t[3],
                              const float* d_xyz, const uint8_t* d_rgba, uint64_t n,
                              int freespace);

/* Counters of the last integrate call (the reference logs some of them through
 * VLOG(3), tsdf_integrator.cc:368-370):
 * [0] normal rays/bundles cast  [1] clearing rays/bundles cast  [2] ray-voxel updates
 * [3] distinct voxels touched   [4] distinct blocks touched     [5] blocks allocated
 * [6] valid points              [7] kernels launched            [8] kernels launched by all
 * integrate calls since vbx_create   [9] / [10] bundles / points folded a second time with IEEE
 * division (diagnostic)   [11] passes the call needed (> 1 when its update records exceed
 * vbx_engine_options.max_updates_per_pass: the synchronous calls then emit and apply contiguous
 * ray ranges one after the other, same result; [3] counts a voxel once per pass)  [12] bits a Merged
 * bundle key uses   [13] asynchronously submitted scans redone synchronously since vbx_create
 * [14] / [15] host time (ns) vbx_tsdf_integrate_async spent waiting for a free hand-off set / enqueueing,
 * summed since vbx_create.
 * After asynchronous submissions: [0..12] are those of the last scan collected (all, after vbx_sync). */
VBX_API int vbx_get_counters(const vbx_ctx* ctx, uint64_t out[16]);
/* Device time (ms, CUDA events on the context's stream) of the last integrate /
 * ESDF update call, excluding host<->device copies of the cloud. */
VBX_API int vbx_last_device_ms(const vbx_ctx* ctx, float* ms);

/* Layer::getNumberOfAllocatedBlocks (core/layer.h:205) */
VBX_API int vbx_num_blocks(vbx_ctx* ctx, int layer, uint64_t* n);
/* Layer::getAllAllocatedBlocks / getAllUpdatedBlocks(bit) (core/layer.h:184-203).
 * updated_mask = 0 lists every block, else only blocks with (updated & mask) != 0.
 * idx3 receives up to cap (x,y,z) triples sorted ascending by (x,y,z); *n = count. */
VBX_API int vbx_list_blocks(vbx_ctx* ctx, int layer, int updated_mask, int32_t* idx3, uint64_t cap,
                    uint64_t* n);
/* Block voxel payloads, device -> host (the lazy host mirror of SURVEY.md N1).
 * voxels: m * vps^3 * sizeof(voxel) bytes; updated_bits: m bytes (may be NULL). */
VBX_API int vbx_download_blocks(vbx_ctx* ctx, int layer, const int32_t* idx3, uint64_t m, void* voxels,
                        uint8_t* updated_bits);
/* The incremental mirror as one call (what a host consumer does after a scan:
 * getAllUpdatedBlocks(bit), core/layer.h:194-203 -> read the blocks -> updated().reset(bit),
 * e.g. mesh_integrator.h:168-183): every block with (updated & updated_mask) != 0 (0 = every
 * block), ascending (x,y,z); payloads are gathered on the device and leave it in ONE copy --
 * directly into `voxels` when that is page-locked (vbx_host_alloc), else through a page-locked
 * staging buffer; clear_mask bits are reset on the device afterwards.
 * *n = number of matching blocks; if *n > cap nothing is copied or cleared (grow and retry). */
VBX_API int vbx_mirror_updated(vbx_ctx* ctx, int layer, int updated_mask, int clear_mask, int32_t* idx3,
                       void* voxels, uint8_t* updated_bits, uint64_t cap, uint64_t* n);
/* The same with payloads in the reference's serialised form (Block::serializeToIntegers,
 * src/core/block.cc:159-183 TSDF = 3 words per voxel, :203-234 ESDF = 2 words per voxel -- the
 * `voxel_data` of BlockProto / voxblox_msgs::Block), packed on the device: words holds
 * cap * vps^3 * (3 | 2) uint32. */
VBX_API int vbx_serialize_updated(vbx_ctx* ctx, int layer, int updated_mask, int clear_mask, int32_t* idx3,
                          uint32_t* words, uint8_t* updated_bits, uint64_t cap, uint64_t* n);
/* ... and back: Block(BlockProto) + deserializeFromIntegers (core/block_inl.h:73-109,
 * block.cc:65-90,110-135); creates the blocks as needed. */
VBX_API int vbx_deserialize_blocks(vbx_ctx* ctx, int layer, const int32_t* idx3, uint64_t m,
                           const uint32_t* words, const uint8_t* updated_bits);
/* Layer files (.vxblx), written from / read into the device map:
 * Layer::saveToFile(file_path, clear_file) (core/layer_inl.h:81-157) and
 * io::LoadBlocksFromFile(file_path, kReplace, multiple_layer_support = true, layer)
 * (io/layer_io_inl.h:13-90): varint message count, LayerProto header, one BlockProto per block
 * (proto/voxblox/*.proto); loaded blocks get every updated bit (layer_inl.h:227).  A file may
 * hold several layers (clear_file = 0 appends); the first compatible one is loaded. */
VBX_API int vbx_save_layer(vbx_ctx* ctx, int layer, const char* path, int clear_file);
VBX_API int vbx_load_layer(vbx_ctx* ctx, int layer, const char* path, uint64_t* n_blocks_loaded);
/* Host-only: the protobuf wire bytes of Layer::getProto / Block::getProto (core/layer_inl.h:41-51,
 * core/block_inl.h:73-109), and the BlockProto parser.  *n = bytes (words) needed; nothing is
 * written if the buffer is too small. */
VBX_API int vbx_proto_encode_layer(double voxel_size, uint32_t voxels_per_side, const char* type, uint8_t* out,
                           uint64_t cap, uint64_t* n);
VBX_API int vbx_proto_encode_block(int32_t voxels_per_side, double voxel_size, const double origin[3], int has_data,
                           const uint32_t* words, uint64_t n_words, uint8_t* out, uint64_t cap, uint64_t* n);
VBX_API int vbx_proto_decode_block(const uint8_t* msg, uint64_t len, int32_t* voxels_per_side, double* voxel_size,
                           double origin[3], int* has_data, uint32_t* words, uint64_t cap_words,
                           uint64_t* n_words);
/* Host -> device: Layer::insertBlock / allocateBlockPtrByIndex + voxel copy
 * (core/layer.h:103-111,152-161); creates the block if needed. */
VBX_API int vbx_upload_blocks(vbx_ctx* ctx, int layer, const int32_t* idx3, uint64_t m,
                      const void* voxels, const uint8_t* updated_bits);
/* Device-to-device block transfer, for keeping read-only replicas of a sharded map's other ranks' blocks
 * (DESIGN.md "multi-GPU").  Both calls take 4-byte aligned DEVICE memory of this context's GPU (cudaMalloc /
 * torch tensors); host and null pointers give VBX_E_INVALID.
 * vbx_gather_updated_device: the gather of vbx_mirror_updated into device memory -- every block with
 * (updated & updated_mask) != 0 (0 = every block), and with owned_only != 0 only the blocks this rank owns
 * (vbx_block_owner), ascending (x,y,z): d_idx3 receives 3 int32 per block, d_voxels the raw voxel payloads
 * (the structs above), and clear_mask bits are reset on the device.  Only the block count reaches the host.
 * *n = number of matching blocks; if *n > cap nothing is copied or cleared (grow and retry). */
VBX_API int vbx_gather_updated_device(vbx_ctx* ctx, int layer, int updated_mask, int clear_mask, int owned_only,
                                      int32_t* d_idx3, void* d_voxels, uint64_t cap, uint64_t* n);
/* vbx_upload_blocks with d_idx3 / d_voxels in device memory: creates the blocks as needed and writes the
 * payloads straight from d_voxels; every written block's updated() bits become `updated_bits` (the reported
 * bits only: VBX_UPDATED_MIRROR stays clear).  The indices (12 B per block) are read back to check them before
 * anything is written.  On a sharded engine (world_size > 1) a block this rank owns gives VBX_E_INVALID and
 * nothing changes: a replica never overwrites the copy of record.  Capacity errors as vbx_upload_blocks. */
VBX_API int vbx_upload_blocks_device(vbx_ctx* ctx, int layer, const int32_t* d_idx3, uint64_t m,
                                     const void* d_voxels, uint8_t updated_bits);
/* Layer::removeBlock / removeAllBlocks (core/layer.h:163-164) */
VBX_API int vbx_remove_blocks(vbx_ctx* ctx, int layer, const int32_t* idx3, uint64_t m);
VBX_API int vbx_clear(vbx_ctx* ctx, int layer);
/* block.updated().reset(bit) over a layer (esdf_integrator.cc:113-121) */
VBX_API int vbx_clear_updated(vbx_ctx* ctx, int layer, int updated_mask);

/* EsdfIntegrator(config, tsdf_layer, esdf_layer) (esdf_integrator.cc:7-22) */
VBX_API int vbx_esdf_create(vbx_ctx* ctx, const vbx_esdf_config* cfg);
/* batch = 0: updateFromTsdfLayer(clear_updated_flag)   (esdf_integrator.cc:104-122)
 * batch = 1: updateFromTsdfLayerBatch()                (esdf_integrator.cc:94-102) */
VBX_API int vbx_esdf_update(vbx_ctx* ctx, int batch, int clear_updated_flag);
/* updateFromTsdfBlocks(tsdf_blocks, incremental = false) (esdf_integrator.h:111-112, cc:124-302):
 * propagate / raise / lower for exactly the listed blocks; indices without a TSDF block are
 * skipped (cc:139-141), an index listed twice is processed once. */
VBX_API int vbx_esdf_update_blocks(vbx_ctx* ctx, const int32_t* idx3, uint64_t m, int incremental);
/* addNewRobotPosition(position) (esdf_integrator.cc:25-92; utils/planning_utils_inl.h:13-62):
 * every unobserved or hallucinated ESDF voxel within clear_sphere_radius of `position` becomes
 * free (+default_distance_m, observed, hallucinated), every still unobserved voxel within
 * occupied_sphere_radius becomes occupied (-default_distance_m); ESDF blocks the spheres reach
 * are allocated (also where the TSDF layer holds no block).  The raise / open queue entries and the
 * updated_blocks_ set this produces are consumed by the next vbx_esdf_update(_blocks), as in
 * the reference.  Counters afterwards: [0] ESDF blocks created [1] voxels set free
 * [2] voxels set occupied [4] raise entries queued [5] open entries queued [7] kernels. */
VBX_API int vbx_esdf_add_robot_position(vbx_ctx* ctx, const float position[3]);
/* EsdfIntegrator::clear() (esdf_integrator.h:135-140): drop what addNewRobotPosition queued */
VBX_API int vbx_esdf_clear(vbx_ctx* ctx);
/* setEsdfMaxDistance / setFullEuclidean / getters (esdf_integrator.h:139-149) */
VBX_API int vbx_esdf_set_max_distance(vbx_ctx* ctx, float max_distance_m);
VBX_API int vbx_esdf_set_full_euclidean(vbx_ctx* ctx, int full_euclidean);
VBX_API int vbx_esdf_get_config(const vbx_ctx* ctx, vbx_esdf_config* out);
/* Counters of the last ESDF update: [0] blocks propagated [1] lower [2] raise [3] new
 * [4] voxels raised [5] wavefront relaxations R [6] wavefront sweeps [7] kernels */
VBX_API int vbx_esdf_get_counters(const vbx_ctx* ctx, uint64_t out[16]);

/* Meshing (SURVEY.md section 8f N3): MeshIntegrator<TsdfVoxel> (mesh/mesh_integrator.h) over the device map.
 * MeshIntegratorConfig (mesh_integrator.h:46-66) minus integrator_threads. */
typedef struct vbx_mesh_config {
  int32_t use_color; /* true  */
  float min_weight;  /* 1e-4  */
} vbx_mesh_config;
/* generateMesh(only_mesh_updated_blocks, clear_updated_flag) (mesh_integrator.h:132-160): marching cubes
 * (mesh/marching_cubes.h:74-164) over every TSDF block, or over those whose Update::kMesh bit is set;
 * clear_updated_flag resets that bit (:171-175).  The meshes stay in device memory until the next
 * call; n_blocks / n_vertices report their size. */
VBX_API int vbx_mesh_generate(vbx_ctx* ctx, const vbx_mesh_config* cfg, int only_mesh_updated_blocks,
                              int clear_updated_flag, uint64_t* n_blocks, uint64_t* n_vertices);
/* The result of the last vbx_mesh_generate: idx3 = 3*n_blocks block indices ascending by (x, y, z);
 * block b owns vertices [first_vertex[b], first_vertex[b+1]) (n_blocks + 1 entries); vertices / normals
 * = 3 floats per vertex in the reference's order (Mesh::vertices / normals, mesh/mesh.h:151-154), colors =
 * r,g,b,a per vertex (only after use_color).  Mesh::indices is 0..n-1 per block
 * (marching_cubes.h:97-99) and is not transferred.  Any pointer may be NULL. */
VBX_API int vbx_mesh_download(vbx_ctx* ctx, int32_t* idx3, uint64_t* first_vertex, float* vertices, float* normals,
                              uint8_t* colors);

/* ICP pose refinement (SURVEY.md section 8f N4): voxblox::ICP (alignment/icp.h:72-233, src/alignment/icp.cc),
 * the optional step in front of integratePointCloud (voxblox_ros/src/tsdf_server.cc:254-299).
 * ICP::Config (icp.h:76-108), field names as spelled there.  num_threads: the reference starts that many
 * racing host threads; the device runs them as `num_threads` warps of one thread block under the
 * round-robin schedule (every round: warp w = 0..T-1 takes the next mini batch, matches it against the
 * pose it saw at its own last successful fusion, fusions applied in warp order) -- one of the schedules
 * the reference's threads can produce, and THE schedule for num_threads = 1.  1 <= num_threads <= 32. */
typedef struct vbx_icp_config {
  int32_t refine_roll_pitch;          /* false */
  int32_t mini_batch_size;            /* 20    */
  float min_match_ratio;              /* 0.8   */
  float subsample_keep_ratio;         /* 0.5   */
  float inital_translation_weighting; /* 100   */
  float inital_rotation_weighting;    /* 100   */
  int32_t num_threads;                /* hardware_concurrency() in the reference */
  int32_t reserved;
} vbx_icp_config;
/* ICP::runICP(tsdf_layer, points, inital_T_tsdf_sensor, &refined_T_tsdf_sensor, seed) (icp.h:118-123,
 * icp.cc:219-259) against the device map: points_C = 3*n floats (host memory), the pose as quaternion
 * (w, x, y, z) + translation.  The point order is randomised exactly as the reference does it
 * (std::shuffle with std::default_random_engine(seed) from the C++ library the engine is built with).
 * *num_updates = the number of mini batches that were fused (the reference's return value).
 * Queued asynchronous scans are drained first: the match runs against the map they produce. */
VBX_API int vbx_icp_run(vbx_ctx* ctx, const vbx_icp_config* cfg, const float* points_C, uint64_t n,
                        const float q_wxyz[4], const float t[3], uint32_t seed, float out_q_wxyz[4], float out_t[3],
                        uint64_t* num_updates);
/* the same with the cloud already in device memory */
VBX_API int vbx_icp_run_device(vbx_ctx* ctx, const vbx_icp_config* cfg, const float* d_points_C, uint64_t n,
                               const float q_wxyz[4], const float t[3], uint32_t seed, float out_q_wxyz[4],
                               float out_t[3], uint64_t* num_updates);

VBX_API int vbx_sync(vbx_ctx* ctx);

/* One map over the GPUs of one box: block-ownership sharding (BASELINE.json north_star; SURVEY.md
 * section 8e "alternative: block-hash ownership (sharded map)"; DESIGN.md "multi-GPU").
 * With vbx_engine_options.world_size = W > 1 every rank receives EVERY scan through the ordinary
 * vbx_tsdf_integrate* calls.  Bundling, the bundle order, the merge and the ray walk are the same
 * deterministic computation on every rank; a rank creates only the blocks it owns
 * (vbx_block_owner(index) == rank) and applies only their voxel updates.  TsdfVoxel updates are
 * order dependent and not associative (tsdf_integrator.cc:205-208), so the shards exchange
 * nothing while integrating: the union of the W shards IS the single-GPU map, bit for bit, and
 * every voxel keeps the reference's one-thread update order.  Consumers either work per shard or
 * gather the blocks they need (vbx_mirror_updated / vbx_upload_blocks on the owner / reader). */
VBX_API int vbx_block_owner(const vbx_ctx* ctx, const int32_t block_index[3], int32_t* owner);

/* Measurement aids (the reference's counterpart is timing::Timer, utils/timing.h:132-199).
 * vbx_timer_start / vbx_timer_stop_ms bracket any number of calls with two CUDA events
 * recorded on the context's stream (device timeline, host gaps included).
 * With stage profiling on, every integrate / ESDF call also records events at its
 * stage boundaries and accumulates per-stage device time:
 *   TSDF  [0] point keys  [1] point sort  [2] ray count + block allocation  [3] scan
 *         [4] slot assign [5] ray emit    [6] update sort                   [7] apply
 *         [8] bundle merge        [12] bundle heads + order
 *   ESDF  [9] propagate   [10] raise      [11] lower wavefront              [13..15] reserved
 * calls[i] counts how many times stage i ran. */
/* Page-locked host buffers for point clouds: vbx_tsdf_integrate copies asynchronously (and at
 * full PCIe rate) only from memory that is page-locked; anything else is staged by the driver.
 * vbx_host_alloc / vbx_host_free wrap cudaHostAlloc / cudaFreeHost; vbx_host_copy_ms times one
 * host->device copy of `bytes` from `src` into the context's staging buffer (diagnostic). */
VBX_API int vbx_host_alloc(vbx_ctx* ctx, size_t bytes, void** out);
VBX_API int vbx_host_free(vbx_ctx* ctx, void* p);
VBX_API int vbx_host_copy_ms(vbx_ctx* ctx, const void* src, size_t bytes, float* ms);
/* Test hooks for the engine's own device primitives (stable radix sort with a device-side
 * element count, exclusive scan); host arrays in, host arrays out. */
VBX_API int vbx_debug_sort(vbx_ctx* ctx, const void* keys, int key_bytes, uint32_t n, int key_bits, void* keys_out,
                   uint32_t* perm_out);
VBX_API int vbx_debug_scan(vbx_ctx* ctx, const uint32_t* in, uint32_t n, uint32_t* out);
/* Test hook for ICP's per-batch arithmetic (the functions vbx_icp_run applies to each mini batch), one
 * device thread per item i < n, row-major 3 x 3 matrices and (w, x, y, z) quaternions:
 *   r_out[9i ..]    the batch rotation of the cross-covariance h[9i ..] (2-D closed form when
 *                   refine_roll_pitch == 0, 3-D SVD otherwise), valid_out[i] = 1 when ICP would fuse it
 *                   (finite and a valid rotation matrix), else 0;
 *   q_out[4i ..]    the quaternion of the rotation matrix m[9i ..];
 *   log_out[3i ..]  the SO(3) log of the quaternion q[4i ..];  exp_out[4i ..] the exp of the vector w[3i ..]. */
VBX_API int vbx_debug_icp_solve(vbx_ctx* ctx, uint32_t n, int refine_roll_pitch, const float* h, const float* m,
                                const float* q, const float* w, float* r_out, int32_t* valid_out, float* q_out,
                                float* log_out, float* exp_out);
/* Test hook: bytes of the page-locked staging buffer that vbx_mirror_updated / vbx_upload_blocks allocate on
 * first use (0 while it has never been allocated). */
VBX_API int vbx_debug_staging_bytes(const vbx_ctx* ctx, uint64_t* host_bytes);
/* Diagnostic for the pipelined path (vbx_tsdf_integrate_async): with the environment variable
 * VBX_ASYNC_TIMELINE set before the first asynchronous submission, the hand-off events keep timestamps.
 * For each of the (at most cap_sets, 10 exist) hand-off sets: seq[k] = submission number of the last scan
 * that used it, ms[5k .. 5k+4] = when its front half started / ended, its ray walk ended, its record sort
 * ended and its apply ended, in ms since the pipeline was created (-1: not recorded).  Call after vbx_sync. */
VBX_API int vbx_debug_async_timeline(vbx_ctx* ctx, uint64_t* seq, float* ms, int cap_sets);
/* Test hook for the Merged integrator's bundle order (the iteration order of the reference's
 * unordered_map voxel_map, tsdf_integrator.cc:318-322, :436-456): element e is the e-th inserted key
 * with LongIndexHash hashes[e]; out[p] = the element at iteration position p.  force_global != 0 uses
 * the global-memory tables even when the shared-memory ones would fit. */
VBX_API int vbx_debug_bundle_order(vbx_ctx* ctx, const uint32_t* hashes, uint32_t n, int force_global, uint32_t* out);
/* Test hook for the TSDF apply (the record sort, k_apply_prep and k_apply of every integrate call):
 * applies n caller-given updates to blocks already in the TSDF layer.  Update r goes to voxel
 * rec_voxel[r] (< voxels_per_side^3) of block idx3[3 * rec_block[r] ..] (rec_block[r] < n_blocks) with
 * the final sdf and weight updateTsdfVoxel uses (tsdf_integrator.cc:186-208) and colour rgba[4r ..];
 * a voxel's updates are applied in the order given, with the config's truncation and max_weight.
 * Block updated() bits are not touched.  VBX_E_INVALID: n > max_updates_per_pass, a block that is
 * not in the TSDF layer or is listed twice, an index out of range.  paths (may be NULL) = the apply-path counts below. */
VBX_API int vbx_debug_apply(vbx_ctx* ctx, const int32_t* idx3, uint32_t n_blocks, uint64_t n, const uint32_t* rec_block,
                            const uint32_t* rec_voxel, const float* sdf, const float* weight, const uint8_t* rgba,
                            uint64_t paths[16]);
/* Counting the apply's paths costs a little on every call, so integrate calls count them only after
 * vbx_debug_count_apply_paths(ctx, 1) (off by default); vbx_debug_apply always counts. */
VBX_API int vbx_debug_count_apply_paths(vbx_ctx* ctx, int enabled);
/* Test hook for the Fast integrator: with enabled != 0 (off by default) later Fast calls walk their rays
 * on one device thread in point order, which is the reference's one-thread schedule, so the approximate
 * sets make the reference's decisions exactly.  Everything after that walk runs as usual.  Slow: for tests only. */
VBX_API int vbx_debug_serial_fast(vbx_ctx* ctx, int enabled);
/* How often each path of the apply ran in the last synchronous integrate call (summed over its passes),
 * the last collected asynchronous scan, or vbx_debug_apply (zero for calls made with counting off): [0] voxel runs longer than 32 updates (one
 * warp each) [1] ... cut short at rest (+T, max_weight) [2..4] 128-record steps decided in one go:
 * weight saturated / integer warp scan / prefix sum [5..8] 32-record chunks decided fast: saturated /
 * unit weights / prefix sum / clamped sequential chain [9] chunks applied update by update [10] runs of
 * at most 32 updates [11] ... that continue past their 256-record tile [12..15] zero. */
VBX_API int vbx_debug_apply_paths(const vbx_ctx* ctx, uint64_t out[16]);
VBX_API int vbx_timer_start(vbx_ctx* ctx);
VBX_API int vbx_timer_stop_ms(vbx_ctx* ctx, float* ms);
VBX_API int vbx_set_stage_profiling(vbx_ctx* ctx, int enabled);
VBX_API int vbx_get_stage_ms(const vbx_ctx* ctx, double ms[16], uint64_t calls[16]);

#ifdef __cplusplus
}
#endif
#endif /* VOXBLOX_B200_H_ */
