/* scannet_b200 — C ABI of the H100-native ScanNet hot path.
 *
 * The reference toolkit exposes NO plugin / operator / FFI interface (SURVEY.md §8b): its
 * seams are three command-line tools and two C++ function/class seams.  Each entry point
 * below names the reference interface it stands in for (paths relative to /root/reference).
 *
 * Conventions: plain C, opaque handles, int status (0 = ok, <0 = error; text via
 * scn_last_error(), thread-local), caller-owned output buffers unless stated, no
 * exceptions cross the boundary, one CUDA stream per handle, handles are not thread-safe.
 * Every compute entry point runs on the GPU; there is no CPU fallback — without a usable
 * CUDA device the call fails with SCN_ERR_CUDA.
 */
#ifndef SCANNET_B200_H
#define SCANNET_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SCN_OK              0
#define SCN_ERR_ARG        -1   /* bad argument */
#define SCN_ERR_CUDA       -2   /* CUDA runtime / no device */
#define SCN_ERR_IO         -3   /* file could not be opened / read / written */
#define SCN_ERR_FORMAT     -4   /* malformed .sens / .ply / .obj / parameter file */
#define SCN_ERR_CAPACITY   -5   /* hash table or block heap exhausted */
#define SCN_ERR_UNSUPPORTED -6  /* e.g. TYPE_OCCI_USHORT depth (needs uplink codec, sensorData.h:711-722) */

const char* scn_last_error(void);
int  scn_version(void);
/* Number of CUDA devices visible (<0 on error). */
int  scn_device_count(void);
/* Creates the CUDA context now (≈0.3 s in a cold process); safe to call from a helper thread while input files are read. */
int  scn_cuda_warmup(void);
/* The batch decoders (scn_inflate_batch_device, scn_jpeg_decode_batch_device) keep their pinned upload slices and device scratch
 * buffers, and scn_fuse_* its frame arrays and its last volume, in per-device pools for the life of the process; this frees the
 * idle ones of the current device. */
int  scn_release_cached_staging(void);
/* Pinned host memory for frame staging (cudaHostAlloc); integrate calls detect it and skip the bounce copy. */
void* scn_host_alloc(size_t bytes);
void  scn_host_free(void* p);
void  scn_free(void* p);                      /* frees buffers this library malloc'ed for the caller */
/* device memory / stream helpers for callers without a CUDA runtime of their own (buffers for scn_sens_decode_depth_device and
 * scn_tsdf_integrate_device); the copies return when the transfer has completed */
void* scn_device_alloc(size_t bytes);
void  scn_device_free(void* p);
int   scn_set_device(int device);                     /* cudaSetDevice for the calling thread (multi-GPU drivers) */
int   scn_device_mem_info(size_t* used_bytes, size_t* total_bytes);
int   scn_stream_create(void** stream_out);          /* non-blocking cudaStream_t */
void  scn_stream_destroy(void* stream);
int   scn_memcpy_h2d(void* d_dst, const void* src, size_t bytes, void* stream);
int   scn_memcpy_d2h(void* dst, const void* d_src, size_t bytes, void* stream);

/* ===================================================================== Segmentator ====
 * Replaces: std::vector<int> segment(const std::string&, float, int)   Segmentator/segmentator.cpp:123
 *           universe* segment_graph(int, int, edge*, float)            Segmentator/segmentator.cpp:71
 *           main / writeToJSON                                         Segmentator/segmentator.cpp:253-288
 */

/* Mesh loading with the same acceptance rules as the reference loader (tinyply path
 * segmentator.cpp:130-140: vertex x,y,z must be 4-byte floats, face list property
 * "vertex_indices" or "vertex_index" with 4-byte indices, triangles only; OBJ path :141-172:
 * original vertices, first shape only).  Buffers are malloc'ed; release with scn_free. */
int scn_mesh_load(const char* path, float** xyz, uint64_t* n_verts, uint32_t** tri, uint64_t* n_faces);

/* flags for scn_segment_mesh */
#define SCN_SEG_DEFAULT        0
#define SCN_SEG_DEVICE_UNIONFIND 1  /* run the Kruskal pass (S5) with the speculative-window device kernel instead of the host loop (default: host; see DESIGN.md §5 for the measured comparison) */
/* test hook (scn_segment_graph only): override introsort's depth limit 2*floor(log2 n) to reach the heap-sort fallback */
#define SCN_SEG_TEST_DEPTH(d)  (((d) & 0xFF) << 8)

/* segment() over raw arrays: seg_out[v] = root vertex id of v's segment, bit-identical to the
 * reference compiled with libstdc++ (incl. std::sort's unstable tie order). */
int scn_segment_mesh(const float* xyz, uint64_t n_verts, const uint32_t* tri, uint64_t n_faces,
                     float k_thresh, int32_t seg_min_verts, int32_t* seg_out, int flags);

/* Intermediates for parity tests: 12-byte {float w; int32 a; int32 b} records, 3 per face,
 * before and after the sort (either pointer may be NULL). */
int scn_segment_mesh_debug(const float* xyz, uint64_t n_verts, const uint32_t* tri, uint64_t n_faces,
                           float k_thresh, int32_t seg_min_verts, int32_t* seg_out, int flags,
                           void* edges_presort, void* edges_sorted, float* vertex_normals,
                           int32_t* roots_after_kruskal);

/* segment_graph(): sorts `edges` (12-byte records) in place exactly like the reference and
 * returns find(v) / size(find(v)) for every vertex after the thresholded Kruskal pass. */
int scn_segment_graph(int32_t n_verts, int64_t n_edges, void* edges, float c,
                      int32_t* roots_out, int32_t* sizes_out, int flags);

/* writeToJSON(): one-line JSON, same byte layout as segmentator.cpp:253-266. */
int scn_write_segs_json(const char* path, const char* scene_id, float k_thresh, int32_t seg_min_verts,
                        const int32_t* seg_indices, uint64_t n);

/* The CLI in library form: `segmentator input.ply [kThresh] [segMinVerts]` (same stdout
 * lines, same output file name <base>.<%f kThresh>.segs.json). Returns the process exit code. */
int scn_segmentator_main(int argc, const char** argv);

/* per-stage timings of the last scn_segment_* call on this thread, milliseconds:
 * [0] H2D, [1] normals, [2] weights, [3] sort, [4] kruskal, [5] small-merge, [6] labels+D2H, [7] total */
int scn_segment_last_timings(float* ms8);
/* rounds taken by the device union-find replay (SCN_SEG_DEVICE_UNIONFIND) in the last scn_segment_mesh call on this thread; 0 = host loop */
uint64_t scn_segment_last_uf_rounds(void);

/* ===================================================================== SensReader =====
 * Replaces: ml::SensorData                                  SensReader/c++/src/sensorData.h:285-1936
 *   ctor/loadFromFile :855,:1250   decompressDepthAlloc :939-946   decompressColorAlloc :929-936
 *   saveToFile :1101-1109          saveToImages :1380-1466         operator<< :1941-1955
 */
typedef struct scn_sens scn_sens;

typedef struct {
  uint32_t version;                 /* 4 */
  uint32_t color_width, color_height, depth_width, depth_height;
  int32_t  color_compression;       /* -1 unknown, 0 raw, 1 png, 2 jpeg   (sensorData.h:346-351) */
  int32_t  depth_compression;       /* -1 unknown, 0 raw u16, 1 zlib u16, 2 occi u16 (:352-357) */
  float    depth_shift;
  uint64_t n_frames, n_imu_frames;
  float    color_intrinsic[16], color_extrinsic[16], depth_intrinsic[16], depth_extrinsic[16];
  char     sensor_name[256];
} scn_sens_info_t;

int  scn_sens_open(const char* path, scn_sens** out);
void scn_sens_close(scn_sens* s);
int  scn_sens_info(const scn_sens* s, scn_sens_info_t* info);
/* camera-to-world (row-major 4x4; all -inf = invalid) + timestamps + compressed sizes */
int  scn_sens_frame_meta(const scn_sens* s, uint64_t frame, float cam2world[16], uint64_t* ts_color,
                         uint64_t* ts_depth, uint64_t* color_bytes, uint64_t* depth_bytes);
/* decoded depth, depth_width*depth_height uint16 (0 = invalid), caller-owned buffer */
int  scn_sens_frame_depth_u16(const scn_sens* s, uint64_t frame, uint16_t* out);
/* decoded colour, color_width*color_height*3 RGB8, caller-owned buffer */
int  scn_sens_frame_color_rgb8(const scn_sens* s, uint64_t frame, uint8_t* out);
/* raw compressed payloads (pointers into the handle; valid until scn_sens_close) */
int  scn_sens_frame_payload(const scn_sens* s, uint64_t frame, const uint8_t** color, const uint8_t** depth);

/* ---- colour decode on the device (R4: sensorData.h:609-616 -> stb_image) ----------------------------------------------
 * n baseline JPEG payloads (host pointers), every one width x height, decoded by the GPU (csrc/jpeg_gpu.cu), byte-identical
 * to scn_sens_frame_color_rgb8 / the reference's stb_image path.
 *   d_lut == NULL : d_out (device) receives n frames of width*height RGB8;
 *   d_lut != NULL : device array of out_px ints = colour pixel index per output pixel (-1 = none -> black); d_out receives n
 *                   frames of out_px RGB8 (colour registered to the depth image, what scn_tsdf_integrate_device consumes).
 * Streams the device path does not handle (progressive, multi-scan, exotic sampling) or flags as corrupt go through the host
 * decoder and are uploaded: same bytes, same errors.  *n_on_device (optional) = frames decoded by the GPU.  `stream` =
 * cudaStream_t (0 = default); returns after the work has completed. */
int scn_jpeg_decode_batch_device(const uint8_t* const* src, const uint64_t* src_bytes, uint32_t n, uint32_t width, uint32_t height,
                                 const int32_t* d_lut, uint32_t out_px, void* d_out, void* stream, uint32_t* n_on_device);
/* timings of the calling thread's last scn_jpeg_decode_batch_device: host parse + pack + upload issue (s), entropy+IDCT kernel (ms), colour kernel (ms) */
int scn_jpeg_last_timings(double* host_s, double* entropy_ms, double* color_ms);
/* colour frames [first, first+n) of an open stream into device memory (JPEG on the GPU; raw / PNG via the host decoder) */
int scn_sens_decode_color_device(const scn_sens* s, uint64_t first, uint32_t n, const int32_t* d_lut, uint32_t out_px, void* d_out,
                                 void* stream, uint32_t* n_on_device);
/* Read-ahead decoder: the counterpart of SensorData::RGBDFrameCacheRead (sensorData.h:1717-1835), which the reconstruction
 * binaries pull frames from.  Background threads (the reference has one; n_threads <= 0 picks min(8, cores)) decode depth and
 * colour of up to cache_size frames ahead of the consumer, in stream order.  scn_sens_cache_next copies the next frame into the
 * caller's buffers (either may be NULL) and returns 1, returns 0 after the last frame, negative on a decode error of that
 * frame.  The scn_sens handle must outlive the cache and must not be modified while it exists. */
typedef struct scn_sens_cache scn_sens_cache;
int  scn_sens_cache_create(const scn_sens* s, uint32_t cache_size, int n_threads, scn_sens_cache** out);
int  scn_sens_cache_next(scn_sens_cache* c, uint16_t* depth_out, uint8_t* color_rgb8_out, uint64_t* ts_depth, uint64_t* ts_color);
void scn_sens_cache_destroy(scn_sens_cache* c);
/* replace a frame's pose (as `recons` writes optimised trajectories back, zParametersScanNet.txt:5) */
int  scn_sens_set_pose(scn_sens* s, uint64_t frame, const float cam2world[16]);
int  scn_sens_save(const scn_sens* s, const char* path);
/* saveToImages(): _info.txt, frame-%06d.color.{jpg,png}, .depth.pgm (P5, 16-bit BE), .pose.txt */
int  scn_sens_save_to_images(const scn_sens* s, const char* out_dir);
/* operator<< text (header summary) into a caller buffer; returns needed length */
int64_t scn_sens_describe(const scn_sens* s, char* buf, uint64_t cap);

/* Writer (initDefault + addFrame + saveToFile pattern, sensorData.h:888-929; Converter/main.cpp:32-41) */
int  scn_sens_create(uint32_t color_w, uint32_t color_h, uint32_t depth_w, uint32_t depth_h,
                     const float color_intrinsic[16], const float depth_intrinsic[16],
                     int32_t color_compression, int32_t depth_compression, float depth_shift,
                     const char* sensor_name, scn_sens** out);
/* colour: raw RGB8 (color_compression 0) or an already-encoded JPEG/PNG payload of color_bytes bytes */
int  scn_sens_add_frame(scn_sens* s, const uint8_t* color, uint64_t color_bytes, const uint16_t* depth,
                        const float cam2world[16], uint64_t ts_color, uint64_t ts_depth);
/* The CLI in library form: `sens <file.sens> [outDir=./out/]` (SensReader/c++/src/main.cpp:28-97). */
int  scn_sens_main(int argc, const char** argv);

/* ===================================================================== TSDF fusion =====
 * Replaces: the external FriedLiver.exe / DepthSensing.exe stage
 *   Server/scan_processor.py:27-35,123-138   (`<exe> <params.txt> <params2.txt> <file.sens>` -> .ply)
 * whose source is NOT in the reference tree.  Numerical spec: DESIGN.md "TSDF spec v1".
 */
typedef struct scn_tsdf scn_tsdf;

typedef struct {
  float    voxel_size;                /* s_SDFVoxelSize               (BASELINE.json: 0.004)           */
  float    trunc_base;                /* s_SDFTruncation                                                */
  float    trunc_scale;               /* s_SDFTruncationScale (m per m of depth)                        */
  float    depth_min, depth_max;      /* s_sensorDepthMin/Max         zParametersScanNet.txt:34-35      */
  float    max_integration_distance;  /* s_SDFMaxIntegrationDistance  :51                               */
  uint32_t weight_sample;             /* s_SDFIntegrationWeightSample :52                               */
  uint32_t weight_max;                /* s_SDFIntegrationWeightMax    :53 (clamped to 255: u8 weight)   */
  uint32_t width, height;             /* integration resolution (BASELINE.json: 640x480)                */
  float    depth_shift;               /* .sens header depthShift (1000)                                 */
  uint64_t hash_slots;                /* open-addressing slots (rounded up to a power of two)           */
  uint64_t max_blocks;                /* 8^3 voxel blocks in the heap (4 KiB each)  s_hashNumSDFBlocks  */
  uint32_t batch_frames;              /* frames fused per block residency, 1..32                        */
  uint32_t flags;                     /* SCN_TSDF_* */
  uint32_t depth_filter;              /* s_depthFilter: bilateral pre-filter of the depth map (zParametersBundlingScanNet.txt:74) */
  float    depth_sigma_d;             /* s_depthSigmaD  (:72) pixels                                    */
  float    depth_sigma_r;             /* s_depthSigmaR  (:73) metres                                    */
} scn_tsdf_params;

#define SCN_TSDF_NO_STATS   1u        /* skip the per-launch counters (N_u, N_b) */
#define SCN_TSDF_KERNEL_TMA    4u     /* always use the cp.async.bulk (TMA) staged integrate kernel (default: only for batches of <= 2 frames) */
#define SCN_TSDF_KERNEL_COLUMN 8u     /* always use the register-resident column kernel */

typedef struct {
  uint64_t frames_integrated, frames_skipped;   /* skipped = invalid (-inf) pose */
  uint64_t blocks_allocated;                    /* live blocks in the heap */
  uint64_t voxels_updated;                      /* Σ_frames N_u */
  uint64_t blocks_visited;                      /* Σ_frames N_b */
  uint64_t algorithmic_bytes;                   /* Σ_frames 2WH + 3WH[colour] + 16 N_u + 16 N_b (SURVEY.md §8d) */
  uint64_t kernel_launches;                     /* kernels this handle launched so far */
  uint32_t error_flags;                         /* bit0 heap full, bit1 table full */
} scn_tsdf_stats_t;

void scn_tsdf_default_params(scn_tsdf_params* p);
/* `key = value;` parameter files as consumed by the external binaries (Server/tools/recons/zParameters*.txt);
 * unknown keys are ignored, known ones override *p. */
int  scn_tsdf_params_from_file(const char* path, scn_tsdf_params* p);
int  scn_tsdf_create(const scn_tsdf_params* p, int device, scn_tsdf** out);
void scn_tsdf_destroy(scn_tsdf* t);
/* Use an existing CUDA stream (cudaStream_t cast to void*; NULL = legacy default stream). */
int  scn_tsdf_set_stream(scn_tsdf* t, void* cuda_stream);
/* One frame from HOST buffers: depth W*H u16, rgb W*H*3 (nullable; must already be registered to
 * the depth image), cam2world row-major 4x4, K = 4x4 depth intrinsic as in the .sens header.
 * Frames whose pose is invalid (cam2world[0] == -inf) are skipped. Asynchronous. */
int  scn_tsdf_integrate(scn_tsdf* t, const uint16_t* depth, const uint8_t* rgb,
                        const float cam2world[16], const float K[16]);
/* n frames from HOST buffers (contiguous frames; poses n*16); H2D copies are pipelined against the
 * kernels.  Identical results to n calls of scn_tsdf_integrate. */
int  scn_tsdf_integrate_batch(scn_tsdf* t, uint32_t n, const uint16_t* depth, const uint8_t* rgb,
                              const float* cam2world, const float K[16]);
/* n frames whose depth/rgb already live in DEVICE memory (poses stay on the host). */
int  scn_tsdf_integrate_device(scn_tsdf* t, uint32_t n, const uint16_t* d_depth, const uint8_t* d_rgb,
                               const float* cam2world, const float K[16]);
int  scn_tsdf_sync(scn_tsdf* t);
int  scn_tsdf_reset(scn_tsdf* t);
int  scn_tsdf_stats(scn_tsdf* t, scn_tsdf_stats_t* out);
/* Optional per-kernel timing: when enabled, CUDA events are recorded on the handle's stream around the
 * alloc and integrate kernels of every batch; scn_tsdf_kernel_times sums them (ms) since enabling.
 * union_blocks = Σ_launches blocks read+written by the integrate kernel (actual 8 KiB/block traffic). */
int  scn_tsdf_profile(scn_tsdf* t, int enable);
int  scn_tsdf_kernel_times(scn_tsdf* t, double* alloc_ms, double* integrate_ms, uint64_t* n_batches,
                           uint64_t* union_blocks);
/* Copies up to `cap` blocks to the host: block_xyz 3*n int32 block coordinates, voxels n*512
 * records of {float sdf; uint8 r,g,b,weight}, x fastest.  Order is heap order (unspecified). */
int  scn_tsdf_download_blocks(scn_tsdf* t, int32_t* block_xyz, void* voxels, uint64_t cap, uint64_t* n);
/* The inverse of scn_tsdf_download_blocks: adds n blocks (same layout, HOST buffers) to the volume, block i at heap
 * index blocks_allocated + i, through the volume's hash so that integration, meshing and reset see them.  Download
 * followed by upload into a fresh volume of the same parameters restores the volume.  Refused with the volume unchanged:
 * a coordinate outside [-2^20, 2^20) or a block given twice or already present (SCN_ERR_ARG), more blocks than
 * max_blocks (SCN_ERR_CAPACITY). */
int  scn_tsdf_upload_blocks(scn_tsdf* t, const int32_t* block_xyz, const void* voxels, uint64_t n);
/* Marching-cubes surface of the current volume (malloc'ed; scn_free).  rgb may be NULL. */
int  scn_tsdf_extract_mesh(scn_tsdf* t, float** xyz, uint8_t** rgb, uint32_t** tri,
                           uint64_t* n_verts, uint64_t* n_faces);
/* PLY writer in the VCGLIB layout Segmentator reads (Server/config/scan_stages.json:33-37). */
int  scn_mesh_save_ply(const char* path, const float* xyz, const uint8_t* rgb, uint64_t n_verts,
                       const uint32_t* tri, uint64_t n_faces);
/* Depth bilateral filter as BundleFusion applies it before integration (zParametersBundlingScanNet.txt:72-74); the only
 * in-tree statement of the kernel is AnnotationTools/Filter2dAnnotations/filter.cu:210-247 (bilateralFilterFloatMapDevice),
 * whose arithmetic (float domain weight, double range weight, -inf = invalid) is reproduced.  depth: w*h uint16 (host);
 * out_metres: w*h float (host), -inf where invalid.  Used inside scn_tsdf_integrate* when params.depth_filter != 0. */
int  scn_depth_bilateral_filter(const uint16_t* depth, uint32_t w, uint32_t h, float depth_shift, float sigma_d, float sigma_r,
                                float* out_metres);
/* ------------------------------------------------------------------------------------------------------------------
 * segs.json consumers (SURVEY.md §8f-4): what the annotation tools do with Segmentator's output.
 * ------------------------------------------------------------------------------------------------------------------ */
/* Reader with the tolerance of AnnotationTools/common/Segmentation.h:57-88: segIndices entries may be JSON ints, uints,
 * strings of digits, or null (-> 0xFFFFFFFF); params.kThresh / params.segMinVerts default to 0 when absent.
 * *seg_out is malloc'ed (release with scn_free); scene_id may be NULL. */
int  scn_segs_load(const char* path, uint32_t** seg_out, uint64_t* n_out, float* k_thresh, uint32_t* seg_min_verts,
                   char* scene_id, size_t scene_id_cap);
/* Segmentation::m_segIdsToVertIds (Segmentation.h:70-75) and computeSurfaceAreaPerSegment (Segmentation.h:113-147) in one pass
 * on the GPU.  Outputs (malloc'ed, scn_free): seg_ids[nS] ascending; vert_offsets[nS+1] + vert_ids[nV]: the vertices of
 * segment k are vert_ids[vert_offsets[k] .. vert_offsets[k+1]) in ascending order (the reference's push_back order);
 * area[nS]: sum of Trianglef::getArea (mLib core-graphics/triangle.h:23-35) over the faces whose three corners all lie in the
 * segment, accumulated in double in ascending face order (the reference adds floats in unordered_map order, so only a
 * tolerance is meaningful).  xyz/tri/area may be NULL/0 to skip the area. */
int  scn_segs_aggregate(const uint32_t* seg, uint64_t n_verts, const float* xyz, const uint32_t* tri, uint64_t n_faces,
                        uint32_t** seg_ids, uint64_t* n_segs, uint64_t** vert_offsets, uint32_t** vert_ids, float** area);
/* Per-vertex object ids from an aggregation (Visualizer.cpp:284-297): group g lists segment ids
 * group_segs[group_offsets[g] .. group_offsets[g+1]); every vertex of those segments gets object id g+1, later groups
 * overwrite earlier ones, vertices of ungrouped segments get 0. */
int  scn_segs_objects_per_vertex(const uint32_t* seg, uint64_t n_verts, const uint32_t* group_segs, const uint64_t* group_offsets,
                                 uint64_t n_groups, uint32_t* obj_out);
/* mLib MeshData::computeVertexNormals (core-mesh/meshData.h:758-782): unit face normals summed per vertex in face order,
 * then normalised with 1/length — bit-identical to the sequential loop. */
int  scn_mesh_vertex_normals(const float* xyz, uint64_t n_verts, const uint32_t* tri, uint64_t n_faces, float* normals_out);
/* Annotation propagation from the decimated to the hi-res mesh (Visualizer::propagateAnnotations, Visualizer.cpp:308-377):
 * for each destination vertex the 3 nearest LABELLED (obj > 0) source vertices decide its object id — the first of them
 * that is closer than maxThresh = max(0.01 * largest source bbox extent, 0.05) and whose normal is within normal_thresh
 * radians wins; otherwise the nearest one's id if all three are within maxThresh and agree; otherwise 0.
 * The reference searches with an approximate FLANN kd-tree; this is the exact 3-NN (ties by source index). */
int  scn_propagate_labels(const float* src_xyz, const float* src_normals, const uint32_t* src_obj, uint64_t n_src,
                          const float* dst_xyz, const float* dst_normals, uint64_t n_dst, float normal_thresh,
                          uint32_t* dst_obj_out);
/* ------------------------------------------------------------------------------------------------------------------
 * GPU depth decode (SURVEY.md §8f-2): TYPE_ZLIB_USHORT payloads (sensorData.h:703-709) are uploaded compressed and inflated
 * in device memory, one warp per frame.  d_depth_out: device pointer, n * depth_width * depth_height uint16, frame after
 * frame — exactly what scn_tsdf_integrate_device consumes.  `stream` is a cudaStream_t (NULL = default stream); the call
 * returns when the frames are decoded.  Same bytes and the same error cases as scn_sens_frame_depth_u16.
 * ------------------------------------------------------------------------------------------------------------------ */
int  scn_sens_decode_depth_device(const scn_sens* s, uint64_t first_frame, uint32_t n, uint16_t* d_depth_out, void* stream);
/* the same for caller-supplied zlib streams: src[i] / src_bytes[i] on the host, each must inflate to >= frame_bytes */
int  scn_inflate_batch_device(const uint8_t* const* src, const uint64_t* src_bytes, uint32_t n, uint64_t frame_bytes, void* d_out,
                              void* stream);
/* timings of the calling thread's last scn_inflate_batch_device: host packing + upload issue (s), kernel (ms, CUDA events), whether
 * the shared-memory-window kernel ran (else the window lives in HBM), streams in the launch */
int  scn_inflate_last_timings(double* pack_s, double* kernel_ms, int* ring_window, uint32_t* n_streams);
/* host build of the same decoder source (one lane): used by the CPU test-suite; not a product path */
int  scn_inflate_host(const uint8_t* src, size_t n, uint8_t* out, size_t cap, size_t* produced);

/* ------------------------------------------------------------------------------------------------------------------
 * Scene fusion driver: .sens -> hashed TSDF -> (optionally) marching cubes -> <out>.ply — the contract of the reference's
 * external reconstruction stage (Server/scan_processor.py:27-35,123-138), one scene per GPU (Server/process.py:75 runs one
 * scan per GPU at a time; SURVEY.md §8e).  decode_mode: NULL = automatic, "gpu" = compressed payloads decoded in HBM,
 * "host" = host thread pool.  A failed scene returns the code of the first call that failed (e.g. SCN_ERR_CAPACITY for a full
 * voxel heap), its text prefixed by the .sens path.
 * ------------------------------------------------------------------------------------------------------------------ */
typedef struct scn_fuse_report {
  int32_t  status;                 /* 0 or the error code of this scene (scn_fuse_many) */
  int32_t  device;
  int32_t  gpu_decode;             /* 1 = payloads were decoded on the GPU */
  uint32_t volume_reused;          /* the pooled volume of the previous scene on this GPU was reset instead of a new one created */
  uint32_t color_frames_on_device; /* JPEG frames the device decoder handled itself (the rest went through the host decoder) */
  uint64_t frames_integrated, frames_skipped, frames_skipped_pose;
  uint64_t blocks_allocated, voxels_updated;
  uint64_t mesh_vertices, mesh_faces;
  uint64_t device_bytes_in_use;    /* cudaMemGetInfo after fusion: volume + decode staging */
  double   fuse_s;                 /* first frame in -> last frame integrated, decode included */
  double   decode_wait_s;          /* of which the integrator waited for the decoders */
  double   depth_decode_s, color_decode_s;   /* busy time of the two decoder threads (overlaps fuse_s) */
  double   integrate_s;            /* integrator: submit + wait for the GPU, all chunks */
  double   depth_pack_s, depth_kernel_s;     /* of depth_decode_s: host packing + upload issue, inflate kernel (CUDA events) */
  double   color_host_s, color_entropy_s, color_convert_s;   /* of color_decode_s: host parse + pack, Huffman+IDCT kernel, colour kernel */
  double   setup_s;                /* open + parse the file, create the volume */
  double   buffers_s, teardown_s;  /* of fuse_s: allocating the double-buffered frame arrays; joining the decoders and freeing them */
  double   mc_s, ply_s, total_s;   /* marching cubes, PLY write, everything incl. opening the file */
} scn_fuse_report_t;
int  scn_fuse_scene(const char* sens_path, const char* out_ply /* NULL: no mesh */, const scn_tsdf_params* params, int device,
                    const char* decode_mode, scn_fuse_report_t* report);
/* n_scenes scenes over n_devices GPUs, one scene per GPU at a time, no data-path collective; reports[i] per scene */
/* sizeof(scn_fuse_report_t) of the library build, for bindings that mirror the struct (tests/test_abi_cpu.py) */
size_t scn_fuse_report_sizeof(void);
int  scn_fuse_many(const char* const* sens_paths, const char* const* out_plys /* NULL or per-scene NULL: no mesh */, uint32_t n_scenes,
                   const scn_tsdf_params* params, const int* devices, uint32_t n_devices, const char* decode_mode,
                   scn_fuse_report_t* reports);
/* `fuse <params.txt> <file.sens> [out.ply]` — the recons/improve stage contract; `fuse --gpus N <params.txt> a.sens b.sens ...` */
int  scn_fuse_main(int argc, const char** argv);

/* ------------------------------------------------------------------------------------------------------------------
 * Mesh cleaning (DESIGN.md §6f): the first step of the `decimate` stage, `meshlabserver -i <id>_vh.ply -o <id>_vh_clean.ply
 * -m vc -s clean.mlx` (Server/scan_processor.py:142-146, Server/tools/meshclean/clean.mlx), stated as mLib's MeshData
 * operators (external/mLib/include/core-mesh/meshData.cpp) and run in clean.mlx's order, every step on the GPU:
 *   1. merge close vertices   mergeCloseVertices(t, approx=false) :217-289, then removeDegeneratedFaces :293-318
 *   2. duplicate faces        removeDuplicateFaces :40-104 (first face of every sorted index triple survives)
 *   3. isolated pieces        removeIsolatedPieces :407-454 + removeIsolatedVertices :324-360 (vertex renumbering by first
 *                             appearance in face/corner order; unreferenced vertices dropped)
 * ------------------------------------------------------------------------------------------------------------------ */
#define SCN_CLEAN_SKIP_MERGE  1u
#define SCN_CLEAN_SKIP_DEDUP  2u
#define SCN_CLEAN_SKIP_PIECES 4u
typedef struct {
  float    merge_threshold;     /* t: vertices closer than t (d^2 < t*t) merge; clean.mlx 0.0010689 */
  uint32_t min_piece_vertices;  /* a face survives only if its piece has >= this many vertices (mLib's unit; 0 = off) */
  uint32_t min_piece_faces;     /* ... and >= this many faces after steps 1-2 (clean.mlx MinComponentSize 7500; 0 = off) */
  uint32_t flags;               /* SCN_CLEAN_SKIP_* */
} scn_mesh_clean_params;
typedef struct scn_mesh_clean_report {
  uint64_t vertices_in, faces_in, vertices_out, faces_out;
  uint64_t vertices_merged;            /* step 1: vertices that mapped onto an earlier representative */
  uint64_t merge_components;           /* step 1: components of >= 2 vertices of the proximity graph (pairs in neighbouring cells, d^2 < t^2) */
  uint64_t largest_merge_component;    /* step 1: vertices in the largest such component (1 when nothing is within t) */
  uint64_t degenerate_faces;           /* step 1: faces with a repeated index after the remap */
  uint64_t duplicate_faces;            /* step 2 */
  uint64_t pieces_total;               /* step 3: pieces with at least one face */
  uint64_t pieces_removed;
  uint64_t faces_in_removed_pieces;
  double   upload_ms, merge_ms, dedup_ms, pieces_ms, download_ms, total_ms;   /* CUDA events on the call's stream */
} scn_mesh_clean_report_t;
void   scn_mesh_clean_default_params(scn_mesh_clean_params* p);
size_t scn_mesh_clean_report_sizeof(void);
/* Reads a MeshLab FilterScript made of clean.mlx's filters (Merge Close Vertices / Remove Duplicate Faces / Remove Isolated
 * pieces (wrt Face Num.) / Remove Unreferenced Vertex, in that order, any of them may be absent): sets merge_threshold,
 * min_piece_faces and the SKIP flags of *p.  Any other filter (e.g. simplify.mlx's Quadric Edge Collapse Decimation) gives
 * SCN_ERR_UNSUPPORTED naming it. */
int  scn_mesh_clean_params_from_mlx(const char* path, scn_mesh_clean_params* p);
/* rgb (n_verts*3) may be NULL; then *rgb_out is NULL.  Outputs are malloc'ed (scn_free); report may be NULL.
 * SCN_ERR_ARG: a face index >= n_verts; unless the merge is skipped also t <= 0 or NaN, a non-finite coordinate, or
 * |v_i / t| >= 2^31 (the cell's int conversion would be undefined). */
int  scn_mesh_clean(const float* xyz, const uint8_t* rgb, uint64_t n_verts, const uint32_t* tri, uint64_t n_faces,
                    const scn_mesh_clean_params* params, float** xyz_out, uint8_t** rgb_out, uint32_t** tri_out,
                    uint64_t* n_verts_out, uint64_t* n_faces_out, scn_mesh_clean_report_t* report);
/* scn_mesh_load plus per-vertex colour: *rgb (n_verts*3, malloc'ed) when the vertex element has uchar red, green and blue,
 * else NULL.  Same acceptance rules as scn_mesh_load. */
int  scn_mesh_load_rgb(const char* path, float** xyz, uint8_t** rgb, uint64_t* n_verts, uint32_t** tri, uint64_t* n_faces);
/* `meshclean -i in.ply -o out.ply [-m vc] [-s script.mlx]`: the meshlabserver arguments of scan_processor.py:143.  Without -s
 * the clean.mlx defaults apply; without `-m vc` the output carries no colour (white). */
int  scn_meshclean_main(int argc, const char** argv);

/* ------------------------------------------------------------------------------------------------------------------
 * Mesh decimation (DESIGN.md §6g): the second and third steps of the `decimate` stage, `meshlabserver -i <id>_vh_clean.ply
 * -o <id>_vh_clean_1.ply -m vc -s simplify.mlx` and again into <id>_vh_clean_2.ply (Server/scan_processor.py:144-145).
 * Quadric edge-collapse decimation (Garland-Heckbert quadrics, binary64) in deterministic rounds of independent collapses,
 * this repository's own spec: MeshLab/VCG is not in the reference tree and the result is NOT MeshLab's mesh.  Then AutoClean
 * (duplicate faces, unreferenced vertices) and the script's clean filters (scn_mesh_clean's steps), every step on the GPU.
 * ------------------------------------------------------------------------------------------------------------------ */
typedef struct {
  uint64_t target_faces;        /* TargetFaceNum: the face target when target_perc == 0 */
  double   target_perc;         /* TargetPerc in [0, 1]: target = floor(faces_in * target_perc) when != 0 (simplify.mlx 0.2) */
  double   quality_thr;         /* QualityThr >= 0: collapses leaving a triangle of quality q < thr cost thr / max(q, 1e-6) times more (0.3) */
} scn_mesh_simplify_params;
typedef struct scn_mesh_simplify_report {
  uint64_t vertices_in, faces_in, vertices_out, faces_out;
  uint64_t target_faces;               /* the face target of the rounds */
  uint64_t rounds;                     /* rounds that applied at least one collapse */
  uint64_t collapses;
  uint64_t faces_collapsed;            /* faces removed by the collapses */
  uint64_t autoclean_duplicate_faces;  /* AutoClean: duplicate faces removed after the rounds */
  uint64_t max_vertex_faces;           /* the largest number of face corners at one vertex, over all rounds */
  double   upload_ms, quadrics_ms, rounds_ms, autoclean_ms, clean_ms, download_ms, total_ms;   /* CUDA events on the call's stream */
  scn_mesh_clean_report_t clean;       /* the clean filters after AutoClean (sizes and counters; all zero when `after` is NULL) */
} scn_mesh_simplify_report_t;
/* simplify.mlx: TargetPerc 0.2, QualityThr 0.3; *after (may be NULL): Merge Close Vertices 0.0010689, Remove Duplicate Faces,
 * Remove Isolated pieces < 1000 faces, Remove Unreferenced Vertex */
void   scn_mesh_simplify_default_params(scn_mesh_simplify_params* p, scn_mesh_clean_params* after);
size_t scn_mesh_simplify_report_sizeof(void);
/* Reads a FilterScript whose first filter is Quadric Edge Collapse Decimation (once) followed by clean.mlx's filters (read as
 * scn_mesh_clean_params_from_mlx does, into *after).  The decimation's booleans must have simplify.mlx's values
 * (OptimalPlacement and AutoClean true, the others false) and BoundaryWeight 1: anything else, an unknown parameter or a script
 * without the decimation gives SCN_ERR_UNSUPPORTED naming it. */
int  scn_mesh_simplify_params_from_mlx(const char* path, scn_mesh_simplify_params* p, scn_mesh_clean_params* after);
/* Shaped like scn_mesh_clean; after == NULL runs no clean filter.  SCN_ERR_ARG: a face index >= n_verts, a non-finite
 * coordinate, target_perc NaN or outside [0, 1], quality_thr NaN or negative, and the refusals of scn_mesh_clean's filters. */
int  scn_mesh_simplify(const float* xyz, const uint8_t* rgb, uint64_t n_verts, const uint32_t* tri, uint64_t n_faces,
                       const scn_mesh_simplify_params* params, const scn_mesh_clean_params* after, float** xyz_out, uint8_t** rgb_out,
                       uint32_t** tri_out, uint64_t* n_verts_out, uint64_t* n_faces_out, scn_mesh_simplify_report_t* report);
/* `meshsimplify -i in.ply -o out.ply [-m vc] [-s simplify.mlx]`: the meshlabserver arguments of scan_processor.py:144-145.
 * Without -s the simplify.mlx defaults apply; without `-m vc` the output carries no colour (white). */
int  scn_meshsimplify_main(int argc, const char** argv);

/* ------------------------------------------------------------------------------------------------------------------
 * Free-space occupancy grid (DESIGN.md §6h): the `freespace` stage, `FreeSpace.exe <id>.sens` -> `<id>.grid`
 * (Server/config/scan_stages.json:43-47, Server/scan_processor.py:150-152).  FreeSpace.exe is not in the reference tree, so the
 * numerics are this repository's own "free-space spec v1" (parity unpinned).  Every voxel of a dense lattice box counts the
 * frames that saw it free (in front of the measured surface) and occupied (inside the band around it); the label is
 * 0 unknown, 1 free, 2 occupied.  Counting runs on the GPU; there is no CPU fallback.
 * ------------------------------------------------------------------------------------------------------------------ */
typedef struct scn_freespace scn_freespace;
typedef struct {
  float    voxel_size;                /* vs, metres (0.05); voxel g has its centre at g*vs                              */
  float    band_base, band_scale;     /* band(d) = fma(band_scale, d, band_base): 0.05 m + 0.01 per metre of depth       */
  float    depth_min, depth_max;      /* valid depth range (0.1 / 6.0 m, zParametersScanNet.txt:34-35)                   */
  float    max_distance;              /* observations end here (4.0 m, zParametersScanNet.txt:51)                        */
  uint64_t max_voxels;                /* capacity of the counted box (2^28 = 2 GiB of counters); larger boxes are refused */
} scn_freespace_params;
typedef struct scn_freespace_report {
  uint64_t frames_used, frames_skipped_pose;   /* frames classified; frames without a pose (cam2world[0] == -inf), never decoded */
  uint64_t envelope_dims[3], output_dims[3];   /* the counted box; the cropped box of labelled voxels (0 when none) */
  int32_t  envelope_lo[3], output_lo[3];
  uint64_t voxels_free, voxels_occupied, voxels_unknown;   /* labels of the output box */
  uint64_t pairs_classified, pairs_culled;     /* (8^3 brick, frame) pairs the classify kernel ran / skipped by the frustum test */
  double   decode_s;                           /* depth decode (GPU inflate or upload), host clock around each call */
  double   classify_ms;                        /* classify kernels, CUDA events */
  double   crop_ms;                            /* label + crop + download, host clock */
  double   write_s, total_s;                   /* .grid write; the whole call incl. opening the file */
} scn_freespace_report_t;
void   scn_freespace_default_params(scn_freespace_params* p);
size_t scn_freespace_report_sizeof(void);
/* The lattice box that holds every voxel the frames can observe, from the poses alone (host only, binary64): the camera centres
 * of the frames with a pose, widened by (max_distance + band(max_distance)) * |(1, (corner - c) / f)| over the image corners
 * +-1 px, plus one voxel, rounded outward.  No frame with a pose: dims 0.  SCN_ERR_ARG: invalid parameters, fx or fy <= 0, a
 * box beyond +-2^23 voxels. */
int  scn_freespace_envelope(const float* cam2world, uint32_t n, const float K[16], uint32_t width, uint32_t height,
                            const scn_freespace_params* p, int32_t lo[3], uint64_t dims[3]);
/* Counts over the box lo .. lo+dims-1 for width x height depth frames.  SCN_ERR_ARG: vs <= 0 or NaN, a band term negative or
 * NaN, depth_min >= depth_max, max_distance <= 0, depth_shift <= 0, frames of 0 or more than 2^24 pixels, a box beyond
 * +-2^23 voxels; SCN_ERR_CAPACITY: a box of more than max_voxels voxels (never truncated). */
int  scn_freespace_create(const scn_freespace_params* p, uint32_t width, uint32_t height, float depth_shift, const int32_t lo[3],
                          const uint64_t dims[3], int device, scn_freespace** out);
void scn_freespace_destroy(scn_freespace* h);
/* n frames, depth n*W*H u16 on the HOST (_integrate) or in DEVICE memory (_integrate_device); poses n*16 row-major cam2world and
 * K (4x4 depth intrinsic as in a .sens header) on the host.  Frames whose pose is invalid (cam2world[0] == -inf) are skipped
 * and their depth is never read.  Counts commute: frame order and the split into calls do not change them.  Returns when the
 * frames are counted.  Host frames travel in one copy per batch on the handle's stream; device frames must be complete when
 * _integrate_device is called (the work that wrote them has finished, as when scn_inflate_batch_device has returned). */
int  scn_freespace_integrate(scn_freespace* h, uint32_t n, const uint16_t* depth, const float* cam2world, const float K[16]);
int  scn_freespace_integrate_device(scn_freespace* h, uint32_t n, const uint16_t* d_depth, const float* cam2world, const float K[16]);
/* The smallest box holding every labelled voxel: labels (u8, x fastest), and optionally the two counts (u32), malloc'ed
 * (scn_free); n_free / n_occ may be NULL.  Empty result: dims 0, lo 0, NULL arrays. */
int  scn_freespace_download(scn_freespace* h, int32_t lo_out[3], uint64_t dims_out[3], uint8_t** labels, uint32_t** n_free,
                            uint32_t** n_occ);
/* What the handle did so far (frames, box, pairs, classify time; output box, label counts and crop time of the last download) */
int  scn_freespace_handle_report(const scn_freespace* h, scn_freespace_report_t* report);
/* .grid file (DESIGN.md §6h): "SCNGRID\0", u32 version 1, f32 vs, u64 dims[3], i32 lo[3], u8 labels x fastest */
int  scn_freespace_save_grid(const char* path, float voxel_size, const int32_t lo[3], const uint64_t dims[3], const uint8_t* labels);
/* The stage: every frame of the .sens with a pose (depth inflated on the GPU) -> envelope -> counts -> labels -> out_grid
 * (NULL: no file).  width, height and depth_shift come from the stream.  report may be NULL. */
int  scn_freespace_scene(const char* sens_path, const char* out_grid, const scn_freespace_params* p, int device,
                         scn_freespace_report_t* report);
/* `freespace [params.txt] <file.sens> [out.grid] [--voxel V]`: writes <base>.grid beside the input unless an output is given.
 * params.txt (scn_tsdf_params_from_file) sets the depth range and max_distance; --voxel V sets voxel_size = band_base = V. */
int  scn_freespace_main(int argc, const char** argv);

/* ------------------------------------------------------------------------------------------------------------------
 * Preview render (DESIGN.md §6i): the `render` stage, `python mts_render.py <id>_vh_clean_2.ply` -> `<id>_vh_clean_2.png`
 * (Server/scan_processor.py:158-160, Server/mts_render.py).  The script path-traces the mesh with Mitsuba, which is not in the
 * reference tree; the numerics here are this repository's own "render spec v1" and the image is NOT Mitsuba's (box-filtered
 * hashed samples, two-sided Lambertian surfaces, no Russian roulette, alpha = coverage).  What the script states is kept: argv,
 * defaults, camera placement, film size, samples, exposure, integrator names and output names.  Tracing runs on the GPU;
 * there is no CPU fallback.
 * ------------------------------------------------------------------------------------------------------------------ */
#define SCN_RENDER_PATH 0             /* constant environment of radiance 1, Lambertian surfaces, max_depth interactions */
#define SCN_RENDER_AO   1             /* one cosine-weighted ray of length ao_length per primary hit: 1 escaped, 0 blocked */
typedef struct {
  uint32_t width, height;             /* film size in pixels (640 x 480), 1 .. 16384 each */
  uint32_t samples;                   /* samples per pixel, 1 .. 256 (16) */
  int32_t  integrator;                /* SCN_RENDER_PATH (default) or SCN_RENDER_AO */
  uint32_t max_depth;                 /* path: surface interactions before a path ends with 0, 1 .. 64 (5) */
  float    exposure;                  /* radiance is scaled by 2^exposure (1.0) */
  float    world_up[3];               /* (0, 0, 1); the turntable axis and the camera's offset direction */
  float    camera_up[3];              /* (0, 1, 0); the image's up vector before lookAt */
  float    camera_offset[3];          /* (0, 0, 0), added to world_up before normalisation (the script leaves its default as is) */
  float    bsphere_mult;              /* camera distance in bounding-sphere radii (2.5) */
} scn_render_params;
/* One view in binary32, made by scn_render_camera.  The sample at film position (fx, fy) (pixel (x, y) covers [x, x+1) x
 * [y, y+1), y down) has direction p00 + fx*du + fy*dv: du and dv are one pixel right and down, and the component of p00
 * along the view axis is 1, so t measures depth along that axis for primary rays. */
typedef struct {
  float origin[3];
  float p00[3];                       /* direction through the top-left corner of the film */
  float du[3], dv[3];
  float t_near;                       /* primary rays count hits with t > t_near (0.01, Mitsuba's default near clip) */
  float t_eps;                        /* secondary rays count hits with t > t_eps (2^-16 r) */
  float ao_length;                    /* length of the ambient-occlusion rays (r, the bounding-sphere radius) */
} scn_render_camera_t;
typedef struct scn_render_report {
  uint64_t views, pixels, samples;    /* per call: views, views*width*height, pixels*samples */
  uint64_t primary_rays, secondary_rays, primary_hits;   /* equal to the oracle's */
  uint64_t node_visits, triangle_tests;                  /* BVH inner nodes entered, ray-triangle tests run */
  uint64_t bvh_nodes;                 /* inner nodes of the tree (faces - 1) */
  double   upload_ms, bvh_ms, trace_ms, download_ms, total_ms;   /* CUDA events on the call's stream; total: host clock */
} scn_render_report_t;
void   scn_render_default_params(scn_render_params* p);
size_t scn_render_report_sizeof(void);
/* The camera of one view, from the axis-aligned box of the n_verts vertices (host only, binary64, rounded once): centre c,
 * radius r = |max - c|, origin = c + bsphere_mult * r * normalize(camera_offset + world_up), lookAt(origin, c, camera_up) with
 * a 45 degree horizontal field of view.  turntable == 0: origin and camera_up rotated by theta degrees about world_up through
 * the world origin (the script's single view); turntable != 0: about the axis through c (its turntable frames).
 * SCN_ERR_ARG: no vertex, a non-finite coordinate, a zero offset + world_up or view direction, camera_up parallel to the
 * view direction, invalid film size. */
int  scn_render_camera(const float* xyz, uint64_t n_verts, const scn_render_params* params, double theta, int turntable,
                       scn_render_camera_t* cam_out);
/* Renders n_views views of the mesh into rgba_out (caller-owned, n_views * height * width * 4 bytes, view-major, rows top
 * down): the BVH is built once on the GPU and every (view, pixel, sample) is traced in one launch.  rgb (n_verts*3, sRGB) may
 * be NULL: reflectance 0.5.  report may be NULL.  SCN_ERR_ARG: no face, a face index >= n_verts, a non-finite coordinate or
 * one of magnitude > 2^28, invalid parameters or cameras; SCN_ERR_CUDA: no device. */
int  scn_render_mesh(const float* xyz, const uint8_t* rgb, uint64_t n_verts, const uint32_t* tri, uint64_t n_faces,
                     const scn_render_params* params, const scn_render_camera_t* cams, uint32_t n_views, uint8_t* rgba_out,
                     scn_render_report_t* report);
/* `render [-o out.png] [--integrator path|ao] [--samples N] [--width W] [--height H] [--theta T] [--exposure E]
 * [--world_up v] [--camera_up v] [--camera_offset v] [--bsphere_mult M] [--render_turntable] [--frames_per_degree D] mesh.ply`:
 * mts_render.py's arguments.  Writes splitext(mesh)[0] + ".png" (or -o), or with --render_turntable the floor(360 / D) frames
 * mesh.ply_000.png ... (D degrees apart; no video).  `mlt` and `vpl` give SCN_ERR_UNSUPPORTED, as does --cameras. */
int  scn_render_main(int argc, const char** argv);

/* ------------------------------------------------------------------------------------------------------------------
 * Camera tracking (DESIGN.md §6j): the tracker of the `recons` stage, `FriedLiver.exe <params.txt> <params2.txt> <id>.sens`
 * (Server/scan_processor.py:27-29,123-126).  BundleFusion is not in the reference tree; this is the repository's own "tracking spec
 * v1", a frame-to-model dense point-to-plane ICP of the kind VoxelHashing's DepthSensing runs (no sparse features, no global
 * optimisation, no relocalisation): NOT BundleFusion's trajectory.  Every frame is tracked against a raycast of the volume, then
 * integrated into it at its tracked pose.  Tracking runs on the GPU; there is no CPU fallback.
 * ------------------------------------------------------------------------------------------------------------------ */
typedef struct scn_track scn_track;
typedef struct {
  uint32_t width, height;             /* tracking / raycast resolution (s_rayCastWidth/Height 320 x 240): the volume's depth
                                         resolution divided by a power of two */
  float    dist_thresh;               /* s_projCorrDistThres (0.15 m): largest |Tp - q| of a pair */
  float    normal_thresh;             /* s_projCorrNormalThres (0.95): smallest n(Tp) . n_q of a pair */
  float    ray_increment_factor;      /* s_SDFRayIncrementFactor (0.8): raycast step in units of the volume's trunc_base */
} scn_track_params;
typedef struct {
  float    cam2world[16];             /* tracked pose; all -inf when the frame was lost (sensorData.h:382) */
  uint32_t iterations[3];             /* Gauss-Newton iterations run per level, finest first */
  uint32_t pairs;                     /* pairs of the last system solved */
  uint32_t valid_pixels;              /* frame pixels with a vertex and a normal at the finest level */
  uint32_t lost;                      /* 1: not integrated, pose invalid */
  double   residual_ss, rms;          /* sum of r^2 of the last system, sqrt(residual_ss / pairs) */
} scn_track_frame_t;
void   scn_track_default_params(scn_track_params* p);
/* `key = value;` parameter files (zParametersScanNet.txt, zParametersBundlingScanNet.txt): the keys above; others are ignored */
int    scn_track_params_from_file(const char* path, scn_track_params* p);
size_t scn_track_frame_sizeof(void);
/* A tracker bound to `vol` (its depth resolution, range, truncation, filter and stream).  SCN_ERR_ARG: a tracking resolution that
 * is not the depth resolution divided by a power of two, or below 12 x 12. */
int    scn_track_create(scn_tsdf* vol, const scn_track_params* p, scn_track** out);
void   scn_track_destroy(scn_track* t);
/* Tracks and integrates n frames whose depth (n * W * H u16) and colour (n * W * H RGB8 registered to the depth image, or NULL)
 * live in DEVICE memory, one after the other: each is tracked against the model of the last integrated frame, then integrated
 * into the volume at its tracked pose and the model is raycast from there.  The first frame of the tracker takes first_pose when
 * it is finite, identity otherwise; later calls continue the same trajectory.  out[i] per frame.  Returns SCN_ERR_CAPACITY when
 * the volume's heap or table ran full. */
int    scn_track_frames(scn_track* t, uint32_t n, const uint16_t* d_depth, const uint8_t* d_rgb, const float K[16], const float first_pose[16],
                        scn_track_frame_t* out);
/* frames tracked and kernels launched so far (tracking, raycast and the volume's integration) */
int    scn_track_stats(const scn_track* t, uint64_t* frames, uint64_t* kernel_launches);
/* GPU time so far by phase, milliseconds from CUDA events on the volume's stream: depth to metres + filter + pyramids + frame maps;
 * the ICP iterations and the pose; the volume's integration; raycast + model maps.  Any pointer may be NULL. */
int    scn_track_phase_ms(const scn_track* t, double* frame_maps_ms, double* icp_ms, double* integrate_ms, double* raycast_ms);

/* The `recons` stage: every frame of the .sens (depth and JPEG colour decoded on the GPU, colour registered as scn_fuse_scene does)
 * tracked and integrated into a new volume, then marching cubes -> out_ply (NULL: no mesh) and the tracked poses (-inf for a lost
 * frame) written into out_sens (NULL: the input, replaced atomically); only the 64-byte pose fields differ from the input.
 * params' width, height and depth_shift come from the stream.  Nothing is written when the call fails (SCN_ERR_IO: the .sens
 * cannot be read; SCN_ERR_CAPACITY: the volume's heap or table ran full; SCN_ERR_ARG: see scn_track_create).  report may be NULL. */
typedef struct scn_recons_report {
  int32_t  status, device;
  uint64_t frames, frames_tracked, frames_lost;
  uint64_t blocks_allocated, mesh_vertices, mesh_faces;
  uint64_t kernel_launches;
  double   setup_s;                    /* open the file, create the volume and the tracker */
  double   recons_s;                   /* first frame decoded -> last frame integrated */
  double   decode_s, track_s;          /* of recons_s: depth + colour decode; tracking + integration (host clock) */
  double   filter_pyramid_ms, icp_ms, integrate_ms, raycast_ms;   /* of track_s: CUDA events (scn_track_phase_ms) */
  double   mc_s, ply_s, sens_s, total_s;   /* marching cubes, PLY write, .sens write, everything */
} scn_recons_report_t;
size_t scn_recons_report_sizeof(void);
int    scn_recons_scene(const char* sens_path, const char* out_ply, const char* out_sens, const scn_tsdf_params* params,
                        const scn_track_params* tparams, int device, scn_recons_report_t* report);
/* `recons <params.txt> <params2.txt> <file.sens> [out.ply]` (the RECONS_BIN contract, Server/scan_processor.py:27-29): both files
 * are read for the volume and the tracker; writes <base>.ply beside the input unless an output is given, and the trajectory into
 * the .sens. */
int    scn_recons_main(int argc, const char** argv);

/* ------------------------------------------------------------------------------------------------------------------
 * Global optimisation of the keyframe trajectory (DESIGN.md §6k, "global optimisation spec v1"): the dense geometric term of
 * BundleFusion's global stage without its sparse features.  Keyframes (one per submap of consecutive frames) are linked by an edge
 * when they are consecutive or when j's depth overlaps i's at the initial poses; every edge contributes point-to-plane residuals
 * between the two keyframes' maps, and Gauss-Newton with block-Jacobi PCG moves every keyframe but the first of each connected
 * component.  Edges whose residual stays high are removed and the solve repeated; a result that still fails is rejected and the
 * poses handed in stand.  Loop closure is the overlap check alone: a revisit is found only when the drifted poses still fall inside
 * the association basin (dist_thresh, normal_thresh).  Everything runs on the GPU; there is no CPU fallback.  `recons --global`
 * (scn_recons_scene_global) runs it inside the `recons` stage.
 * ------------------------------------------------------------------------------------------------------------------ */
typedef struct scn_globalopt scn_globalopt;
typedef struct {
  uint32_t submap_size;               /* s_submapSize (10): frames per submap; its first tracked frame is the keyframe */
  uint32_t max_keyframes;             /* s_maxNumImages (2000), at most 65535 (one grid row of the overlap check per keyframe) */
  uint32_t width, height;             /* s_downsampledWidth/Height (80 x 60): the depth resolution divided by a power of two */
  float    dist_thresh;               /* s_denseDistThresh (0.15 m) */
  float    normal_thresh;             /* s_denseNormalThresh (0.95) */
  float    depth_min, depth_max;      /* s_denseDepthMin/Max (0.5, 4.0 m): the range test of the keyframe depth */
  uint32_t overlap_subsample;         /* s_denseOverlapCheckSubsampleFactor (4) */
  uint32_t nonlin_iters;              /* s_numGlobalNonLinIterations (3), at most 16 */
  uint32_t lin_iters;                 /* s_numGlobalLinIterations (150) */
  float    verify_thresh;             /* s_verifyOptErrThresh (0.05 m): largest edge RMS at the final poses */
  uint32_t max_removed;               /* s_maxNumResidualsRemoved (10) */
} scn_globalopt_params;
typedef struct {
  uint32_t keyframes, edges_consecutive, edges_loop, edges_removed, rejected;
  uint32_t solves;                    /* 1 + edges removed */
  uint32_t nonlin_iterations, lin_iterations;   /* Gauss-Newton and PCG iterations run over all solves */
  uint64_t pairs_before, pairs_after; /* pairs over the edges at the poses handed in / at the final poses */
  double   rss_before, rss_after, rms_before, rms_after;
  double   max_edge_rms;              /* largest edge RMS at the final poses */
  double   rss_iter[16];              /* sum of r^2 at the start of each Gauss-Newton iteration of the last solve */
  double   keyframe_maps_ms, overlap_ms, linearise_ms, pcg_ms, verify_ms;   /* GPU time, CUDA events */
} scn_globalopt_report_t;
typedef struct {
  uint32_t i, j, loop, removed;       /* loop: not consecutive keyframes; removed by verification */
  uint32_t pairs;                     /* at the final poses (0 once removed) */
  uint32_t pad_;
  double   rss, rms;
} scn_globalopt_edge_t;
void   scn_globalopt_default_params(scn_globalopt_params* p);
/* `key = value;` parameter files (zParametersBundlingScanNet.txt): the keys above; others are ignored */
int    scn_globalopt_params_from_file(const char* path, scn_globalopt_params* p);
size_t scn_globalopt_report_sizeof(void);
/* An optimiser bound to `vol` (its depth resolution, depth shift, filter and stream).  SCN_ERR_ARG: a keyframe resolution that is not
 * the depth resolution divided by a power of two, or below 3 x 3, or other parameters out of range. */
int    scn_globalopt_create(scn_tsdf* vol, const scn_globalopt_params* p, scn_globalopt** out);
void   scn_globalopt_destroy(scn_globalopt* g);
/* Adds n keyframes whose depth (n * W * H u16) lives in DEVICE memory and whose cam2world poses (n * 16) are on the host; K is the
 * depth intrinsic.  SCN_ERR_CAPACITY when the keyframes would exceed max_keyframes (none of the n is added). */
int    scn_globalopt_add_keyframes(scn_globalopt* g, uint32_t n, const uint16_t* d_depth, const float* poses, const float K[16]);
/* Solves the keyframes added so far: poses_out (keyframes * 16) receives the optimised cam2world, or the poses handed in when the
 * result is rejected.  report may be NULL. */
int    scn_globalopt_solve(scn_globalopt* g, float* poses_out, scn_globalopt_report_t* report);
/* The edges of the last solve in (i, j) order: writes min(n, cap) entries and the edge count to *n. */
int    scn_globalopt_edges(const scn_globalopt* g, scn_globalopt_edge_t* out, uint32_t cap, uint32_t* n);
/* The `recons` stage with the global optimisation (`recons --global`): scn_recons_scene's tracking, and each chunk's keyframes (the
 * first tracked frame of every submap of gparams->submap_size frames) handed to an optimiser on the tracking volume.  After the
 * last chunk the keyframes are solved; every other tracked frame follows its submap's keyframe, T_f' = T_k' (T_k^-1 T_f) in binary64
 * rounded once (lost frames keep -inf); the stream is re-integrated at the new poses into a fresh volume by scn_fuse_scene's driver
 * (its batch size and decode, params as given), out_ply is written from that volume and then the poses into out_sens.  A rejected
 * result leaves the output of scn_recons_scene.  Nothing is written when the call fails (SCN_ERR_CAPACITY also for more keyframes
 * than gparams->max_keyframes).  report and greport may be NULL. */
int    scn_recons_scene_global(const char* sens_path, const char* out_ply, const char* out_sens, const scn_tsdf_params* params,
                               const scn_track_params* tparams, const scn_globalopt_params* gparams, int device, scn_recons_report_t* report,
                               scn_globalopt_report_t* greport);

#ifdef __cplusplus
}
#endif
#endif /* SCANNET_B200_H */
