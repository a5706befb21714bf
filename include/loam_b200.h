/* loam_b200.h -- C ABI of libloam_b200.so: the B200 (sm_100a) implementation of LOAM's per-sweep registration hot
 * path behind the reference's Basic* classes (laboshinl/loam_velodyne).
 *
 * Plain pointers and sizes only.  Every entry point returns 0 on success or a negative loam_b200_status; nothing
 * throws across this boundary.  A context owns one device, one stream and all device memory; it is not thread-safe
 * (the reference classes are used from one thread each, e.g. LaserOdometry.cpp:254-270) but several contexts may
 * coexist.  Unless stated otherwise host buffers are only read/written during the call (the call synchronises its
 * stream before returning), so callers may reuse them immediately.
 *
 * Points are packed float[4] = (x, y, z, intensity); indices are int32 (nanoflann_pcl.h:102).
 * "Too few points / too few correspondences" are results, not errors: they are reported through counts so the
 * caller can mirror the reference's `continue`s (BasicLaserOdometry.cpp:484-488, BasicLaserMapping.cpp:826-828).
 */
#ifndef LOAM_B200_H
#define LOAM_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct loam_b200_ctx loam_b200_ctx;

typedef enum {
  LOAM_B200_OK = 0,
  LOAM_B200_ERR_ARG = -1,      /* null pointer / negative size / inconsistent ranges */
  LOAM_B200_ERR_CUDA = -2,     /* a CUDA runtime call failed; loam_b200_last_error() has the text */
  LOAM_B200_ERR_NO_DEVICE = -3,/* no CUDA device / device is not sm_90 */
  LOAM_B200_ERR_STATE = -4,    /* call sequence violated (e.g. iterate before set) */
  LOAM_B200_ERR_CAPACITY = -5, /* caller-provided output capacity too small */
  LOAM_B200_ERR_COMM = -6      /* NCCL failure, or a peer of the cube-sharded map did not answer (fused all-reduce) */
} loam_b200_status;

const char* loam_b200_strerror(int status);
/* text of the last CUDA/NCCL failure seen by this context (empty string if none) */
const char* loam_b200_last_error(const loam_b200_ctx* ctx);
/* library version: major*10000 + minor*100 + patch */
int loam_b200_version(void);

/* Create a context on CUDA device `device` (>= 0).  Fails with LOAM_B200_ERR_NO_DEVICE when there is no usable GPU:
 * there is deliberately no CPU fallback. */
int loam_b200_create(loam_b200_ctx** out, int device);
int loam_b200_destroy(loam_b200_ctx* ctx);
/* Scheduling priority of the context's streams relative to other contexts on the same GPU: level 0 = default, 1 = high
 * (the latency-critical Gauss-Newton loops of the odometry stage), -1 = low.  Call right after loam_b200_create, before
 * any work has been enqueued (the streams are re-created). */
int loam_b200_set_priority(loam_b200_ctx* ctx, int level);
/* ---- multi-GPU with the map sharded by cube slabs (SURVEY.md section 8e; csrc/shard.cuh, csrc/peer.inc) --------------------
 * One process per GPU.  Rank r owns the slabs of `slab_cells` 1 m cells along x with (slab index mod world) == r and stores a
 * 2-cell halo around them; it evaluates the scan-to-map queries whose transformed position falls into a cell it owns, and the
 * 32 partial sums of every Gauss-Newton iteration are all-reduced INSIDE the iteration kernel: the folding CTA stores them
 * into every peer's inbox over NVLink (CUDA IPC mapped memory), flags them, and adds the world contributions in rank order,
 * so every rank holds bit-identical normal equations without a host round trip or a separate collective.
 *   loam_b200_peer_export   -> this rank's inbox as a 64-byte CUDA IPC handle (distribute with any all-gather)
 *   loam_b200_peer_connect  <- world x 64 bytes of handles in rank order
 *   loam_b200_peer_connect_local: the same wiring for contexts of ONE process (tests, single-process multi-GPU)
 * After connecting: loam_b200_map_pool_append / seedMap must only be given the points this rank stores
 * (loam_b200_shard_stores), inserted points are filtered by the library; loam_b200_map_iterate returns the all-reduced sums.
 * Every rank must run the same sequence of sweeps and iterations (they do: same sums, same solve). */
int loam_b200_peer_export(loam_b200_ctx* ctx, unsigned char handle_out[64]);
int loam_b200_peer_connect(loam_b200_ctx* ctx, int rank, int world, const unsigned char* handles, int slab_cells);
int loam_b200_peer_connect_local(loam_b200_ctx** ctxs, int world, int slab_cells);
int loam_b200_peer_disconnect(loam_b200_ctx* ctx);
/* host logic of the slab partition: owner of the cell with x index cell_x; does `rank` store the point with coordinate x */
int loam_b200_shard_owner(int cell_x, int slab_cells, int world);
int loam_b200_shard_stores(float x, int rank, int world, int slab_cells);
/* The library records some per-sweep enqueue sequences by stream capture and launches them as one graph.  While a stream
 * records, cudaDeviceSynchronize() from any thread of the process returns an error, so the sequence issued by the context's
 * helper thread (the asynchronous end-of-sweep map update) is only recorded after the caller has opted in here -- i.e. has
 * promised to synchronise through loam_b200_sync / loam_b200_pipeline_sync (or per stream) rather than device-wide while
 * sweeps are in flight.  The streaming pipeline (loam_b200_pipeline_submit) opts in.  LOAM_B200_NO_CAPTURE=1 disables all
 * recording. */
int loam_b200_allow_async_capture(loam_b200_ctx* ctx, int on);
/* Bind the calling host thread to a CUDA device (cudaSetDevice): every host thread other than the one that created a
 * context must call this once before using the context (helper threads of the library do so themselves). */
int loam_b200_bind_thread(int device);
int loam_b200_sync(loam_b200_ctx* ctx);
/* cudaStream_t of the context (as void*) so callers can order their own work / time with events */
void* loam_b200_stream(loam_b200_ctx* ctx);

/* ------------------------------------------------------------------------------------------------------------------
 * Scan registration: replaces BasicScanRegistration::extractFeatures with setScanBuffersFor / setRegionBuffersFor /
 * markAsPicked (BasicScanRegistration.cpp:155-254, 284-386) including the per-ring VoxelGrid of the less-flat points
 * (:246-252).  Parameter names follow RegistrationParams (BasicScanRegistration.h:37-71).
 * ------------------------------------------------------------------------------------------------------------------ */
typedef struct {
  int nFeatureRegions;              /* 6  */
  int curvatureRegion;              /* 5  */
  int maxCornerSharp;               /* 2  */
  int maxCornerLessSharp;           /* 20 */
  int maxSurfaceFlat;               /* 4  */
  float lessFlatFilterSize;         /* 0.2 */
  float surfaceCurvatureThreshold;  /* 0.1 */
} loam_b200_reg_params;

typedef struct {
  /* picks in the reference's output order (ring-major, region-major, pick order), as indices into the input cloud */
  int32_t* sharp_idx;       int sharp_cap;       int n_sharp;
  int32_t* less_sharp_idx;  int less_sharp_cap;  int n_less_sharp;
  int32_t* flat_idx;        int flat_cap;        int n_flat;
  /* per-point label, n entries: 2 sharp, 1 less sharp, 0 less flat, -1 flat (PointLabel, BasicScanRegistration.h:24-30),
   * 127 = not inside any feature region.  May be NULL. */
  int8_t* label;
  /* voxel-filtered less-flat cloud (ring-major; within a ring ascending voxel index, like pcl::VoxelGrid) */
  float* less_flat_ds;      int less_flat_cap;   int n_less_flat;
} loam_b200_features;

/* pts: n packed points, ring-ordered; ring_start/ring_end: the inclusive IndexRange of each ring exactly as
 * processScanlines builds _scanIndices (BasicScanRegistration.cpp:38-41), so empty rings are (c, c-1) or (0, 0).
 * Limits the reference does not have (a ring is staged in one CTA's shared memory): a ring longer than 5344 points
 * returns LOAM_B200_ERR_CAPACITY; curvatureRegion > 15 or nFeatureRegions > 4095 return LOAM_B200_ERR_ARG; the ring
 * binning front end (loam_b200_reg_bin) takes at most 254 rings.  (HDL-64E: 2.1 k points per ring at 10 Hz; the
 * limits are repeated in INTEGRATION.md.) */
int loam_b200_extract_features(loam_b200_ctx* ctx, const float* pts, int n, const int32_t* ring_start,
                               const int32_t* ring_end, int n_rings, const loam_b200_reg_params* params,
                               loam_b200_features* out);

/* ------------------------------------------------------------------------------------------------------------------
 * k-NN search structure: replaces nanoflann::KdTreeFLANN<PointXYZI>::setInputCloud / nearestKSearch
 * (nanoflann_pcl.h:131-152; nanoflann.hpp:1217-1262, 1354-1412) with a Morton-sorted linear BVH held in HBM.
 * Slots: the reference keeps four trees alive (last corner / last surface in odometry, corner / surface map in
 * mapping, BasicLaserOdometry.h:83-84, BasicLaserMapping.cpp:623-624).
 * ------------------------------------------------------------------------------------------------------------------ */
enum { LOAM_B200_TREE_ODOM_CORNER = 0, LOAM_B200_TREE_ODOM_SURF = 1, LOAM_B200_TREE_MAP_CORNER = 2,
       LOAM_B200_TREE_MAP_SURF = 3, LOAM_B200_NUM_TREES = 4 };

/* upload m points and (re)build the tree of `slot`; m may be 0 */
int loam_b200_tree_build(loam_b200_ctx* ctx, int slot, const float* pts, int m);
int loam_b200_tree_size(loam_b200_ctx* ctx, int slot);
/* exact k nearest neighbours (k <= 8) of nq queries (packed float[4], intensity ignored), ascending squared distance,
 * float L2 accumulated x->y->z like nanoflann's L2_Simple_Adaptor (nanoflann.hpp:372-379).  Only points with
 * d2 < max_d2 are reported (pass INFINITY for the plain search); missing neighbours have idx -1 and d2 = FLT_MAX. */
int loam_b200_tree_knn(loam_b200_ctx* ctx, int slot, const float* queries, int nq, int k, float max_d2,
                       int32_t* idx_out, float* d2_out);

/* ------------------------------------------------------------------------------------------------------------------
 * Scan-to-map Gauss-Newton iteration: replaces the body of the iteration loop of
 * BasicLaserMapping::optimizeTransformTobeMapped up to and including AtA / AtB
 * (BasicLaserMapping.cpp:665-866: pointAssociateToMap, 5-NN, line / plane fit, residual weight, Jacobian rows,
 * normal equations).  The 6x6 solve and pose update stay with the caller (:867-922).
 * ------------------------------------------------------------------------------------------------------------------ */
/* DS corner / surface stacks of this sweep (BasicLaserMapping.cpp:519-527), sensor frame */
int loam_b200_map_set_queries(loam_b200_ctx* ctx, const float* corner, int n_corner, const float* surf, int n_surf);

typedef struct {
  float rot[3];   /* rot_x, rot_y, rot_z of _transformTobeMapped */
  float sin_[3];  /* Angle::sin() of the three, as cached by the host (Angle.h:23-26) */
  float cos_[3];
  float pos[3];
} loam_b200_pose;

typedef struct {
  float AtA[36];      /* row-major 6x6, columns (rot_x, rot_y, rot_z, x, y, z) */
  float AtB[6];
  int n_selected;     /* laserCloudSelNum (BasicLaserMapping.cpp:826) */
  int n_corner_selected;
} loam_b200_normal_eq;

int loam_b200_map_iterate(loam_b200_ctx* ctx, const loam_b200_pose* pose, loam_b200_normal_eq* out);
/* debug / parity variant: additionally returns per query (corner queries first, then surface) the coefficient
 * (s*n, s*d) of _coeffSel and a selected flag; coeff: (n_corner+n_surf) x 4 floats, selected: (n_corner+n_surf) */
int loam_b200_map_iterate_debug(loam_b200_ctx* ctx, const loam_b200_pose* pose, loam_b200_normal_eq* out,
                                float* coeff, int8_t* selected);

/* instrumented variant: same result plus the number of grid-table probes (16 B each) and candidate map points (16 B
 * each) the 5-NN searches of this launch read (feeds the algorithmic-bytes figure of the roofline); slower, never
 * used on the timed path */
int loam_b200_map_iterate_stats(loam_b200_ctx* ctx, const loam_b200_pose* pose, loam_b200_normal_eq* out,
                                unsigned long long* table_probes, unsigned long long* candidate_points);

/* ------------------------------------------------------------------------------------------------------------------
 * Scan-to-scan Gauss-Newton iteration: replaces the body of the iteration loop of BasicLaserOdometry::process up to
 * AtA / AtB (BasicLaserOdometry.cpp:246-557: transformToStart, 1-NN + adjacent-ring search every 5th iteration,
 * point-to-line / point-to-plane residuals, Jacobian rows, normal equations).
 * ------------------------------------------------------------------------------------------------------------------ */
/* last less-sharp / less-flat clouds (already transformed to the sweep end, integer-ring intensities) */
int loam_b200_odom_set_last(loam_b200_ctx* ctx, const float* corner, int n_corner, const float* surf, int n_surf);
/* current sharp / flat feature clouds (intensity = ring + relTime) */
int loam_b200_odom_set_current(loam_b200_ctx* ctx, const float* sharp, int n_sharp, const float* flat, int n_flat);

typedef struct {
  float rot[3];
  float sin_[3];
  float cos_[3];
  float pos[3];
  float inv_scan_period; /* 1.f / _scanPeriod (BasicLaserOdometry.cpp:42) */
  int iter;              /* iterCount: search on iter % 5 == 0, weights on iter >= 5 */
} loam_b200_odom_pose;

int loam_b200_odom_iterate(loam_b200_ctx* ctx, const loam_b200_odom_pose* pose, loam_b200_normal_eq* out);
/* debug: coefficient + selected flag per query (sharp first, then flat) and the correspondence indices
 * (ind: (n_sharp+n_flat) x 3 ints: closest, second, third (-1 when absent)) */
int loam_b200_odom_iterate_debug(loam_b200_ctx* ctx, const loam_b200_odom_pose* pose, loam_b200_normal_eq* out,
                                 float* coeff, int8_t* selected, int32_t* ind);

/* ------------------------------------------------------------------------------------------------------------------
 * Whole Gauss-Newton loops with the pose kept on the device: replace the iteration LOOPS of
 * BasicLaserOdometry::process (BasicLaserOdometry.cpp:246-622: correspondences every 5th iteration, normal equations,
 * `continue` below 10 selected points, colPivHouseholderQr solve, degeneracy projection of the first iteration, pose
 * update, non-finite reset, deltaR / deltaT abort) and of BasicLaserMapping::optimizeTransformTobeMapped
 * (BasicLaserMapping.cpp:646-922, `continue` below 50, eigenvalue threshold 100).  Same arithmetic as the
 * per-iteration entry points + a host solve, except that the sin / cos of the updated angles come from the device
 * (double sincos rounded once instead of the host's float libm).  Queries / last clouds / map as for *_iterate.
 * loam_b200_map_solve returns LOAM_B200_ERR_STATE when a shard or communicator is set (use loam_b200_map_iterate).
 * ------------------------------------------------------------------------------------------------------------------ */
typedef struct {
  float rot[3];     /* optimised rot_x, rot_y, rot_z */
  float pos[3];
  int iterations;   /* iterCount + 1 of the last executed iteration (0 when nothing ran) */
  int converged;    /* loop ended (abort thresholds met or iteration cap reached) */
} loam_b200_lm_result;
int loam_b200_odom_solve(loam_b200_ctx* ctx, const float rot[3], const float pos[3], float inv_scan_period,
                         int max_iterations, float delta_t_abort, float delta_r_abort, loam_b200_lm_result* out);
int loam_b200_map_solve(loam_b200_ctx* ctx, const float rot[3], const float pos[3], int max_iterations,
                        float delta_t_abort, float delta_r_abort, loam_b200_lm_result* out);

/* Test hook: the warp-parallel 6 x 6 Gauss-Newton step of the device-resident loops (csrc/lmstep_warp.cuh) on n systems
 * given as 42 floats each (AtA row-major 36, AtB 6) -> x_out (6 per system), degenerate_out (0 / 1 per system).  Must equal
 * loam_b200_host_gn_solve (include/loam_b200_host.h) bit for bit. */
int loam_b200_debug_gn_solve(loam_b200_ctx* ctx, const float* ata_atb, int n, int first_iteration, float eigen_threshold,
                             float* x_out, int* degenerate_out);

/* Test hook: the radix sort every stage shares (8 bits per pass, min(ceil(key_bits / 8), 4) passes) on n host pairs.
 * n_live >= 0 is passed as the sort's device-side live count (only the first min(n, n_live) pairs are sorted and
 * returned meaningfully); n_live < 0 passes none.  out_params == 0 sorts as the callers that read the first buffer
 * directly (an even number of passes).  keys_out / vals_out receive n entries; *path_out the path that ran: 0 the
 * one-cluster sort (0 < n <= 131072 and clusters usable), 1 onesweep with 4 items per thread (n < 200000), 2 onesweep
 * with 16, -1 nothing (n == 0).  LOAM_B200_ERR_ARG for a NULL pointer, n < 0 or key_bits outside 1..32. */
int loam_b200_debug_sort_pairs(loam_b200_ctx* ctx, const uint32_t* keys, const int32_t* vals, int n, int n_live,
                               int key_bits, int out_params, uint32_t* keys_out, int32_t* vals_out, int* path_out);

/* BasicLaserOdometry::transformToEnd (BasicLaserOdometry.cpp:57-87) without IMU terms, in place on n host points */
int loam_b200_transform_to_end(loam_b200_ctx* ctx, float* pts, int n, const loam_b200_odom_pose* pose);
/* pointAssociateToMap over n host points in place (BasicLaserMapping.cpp:207-219, 235-240) */
int loam_b200_transform_to_map(loam_b200_ctx* ctx, float* pts, int n, const loam_b200_pose* pose);

/* pcl::VoxelGrid<PointXYZI> centroid filter (call sites BasicLaserMapping.cpp:519-527,580-588): writes at most
 * cap points, ascending voxel index; *n_out receives the count. */
int loam_b200_voxel_grid(loam_b200_ctx* ctx, const float* pts, int n, float leaf, float* out, int cap, int* n_out);

/* ------------------------------------------------------------------------------------------------------------------
 * Device-resident stage API.  The Basic* drop-in classes keep their clouds in HBM between calls and only
 * materialise a pcl::PointCloud on the host when an accessor is used; these are the entry points they call.  Clouds
 * live in numbered slots of a context; each class owns a disjoint range of slots.
 * ------------------------------------------------------------------------------------------------------------------ */
enum {
  /* BasicScanRegistration outputs (BasicScanRegistration.h:156-163) */
  LOAM_B200_C_REG_FULL = 0, LOAM_B200_C_REG_SHARP, LOAM_B200_C_REG_LESS_SHARP, LOAM_B200_C_REG_FLAT, LOAM_B200_C_REG_LESS_FLAT,
  /* BasicLaserOdometry inputs / outputs (BasicLaserOdometry.h:22-31) */
  LOAM_B200_C_ODOM_SHARP, LOAM_B200_C_ODOM_LESS_SHARP, LOAM_B200_C_ODOM_FLAT, LOAM_B200_C_ODOM_LESS_FLAT, LOAM_B200_C_ODOM_FULL,
  LOAM_B200_C_ODOM_LAST_CORNER, LOAM_B200_C_ODOM_LAST_SURF,
  /* BasicLaserMapping inputs / internals / outputs (BasicLaserMapping.h:88-90,150-162) */
  LOAM_B200_C_MAP_CORNER_LAST, LOAM_B200_C_MAP_SURF_LAST, LOAM_B200_C_MAP_FULL, LOAM_B200_C_MAP_CORNER_STACK_DS,
  LOAM_B200_C_MAP_SURF_STACK_DS, LOAM_B200_C_MAP_CORNER_FROM_MAP, LOAM_B200_C_MAP_SURF_FROM_MAP, LOAM_B200_C_MAP_SURROUND_DS,
  LOAM_B200_C_MAP_CORNER_POOL, LOAM_B200_C_MAP_SURF_POOL,
  LOAM_B200_NUM_CLOUDS
};

int loam_b200_cloud_upload(loam_b200_ctx* ctx, int slot, const float* pts, int n);
/* d_pts: DEVICE pointer to n packed points (e.g. a torch tensor); device-to-device copy on the context's stream */
int loam_b200_cloud_upload_device(loam_b200_ctx* ctx, int slot, const void* d_pts, int n);
int loam_b200_cloud_download(loam_b200_ctx* ctx, int slot, float* out, int cap, int* n_out);
int loam_b200_cloud_size(loam_b200_ctx* ctx, int slot);
int loam_b200_cloud_swap(loam_b200_ctx* ctx, int slot_a, int slot_b);
/* copy a cloud between slots, possibly of two different contexts on the same device (stream-ordered, no host hop) */
int loam_b200_cloud_copy(loam_b200_ctx* dst_ctx, int dst_slot, loam_b200_ctx* src_ctx, int src_slot);
/* count copies dst[i] <- src[i] with one stream hand-shake per direction */
int loam_b200_cloud_copy_many(loam_b200_ctx* dst_ctx, const int* dst, loam_b200_ctx* src_ctx, const int* src, int count);

/* Ring-binning front end = MultiScanRegistration::process up to the processScanlines call
 * (MultiScanRegistration.cpp:160-238, mapper :44-67): n unordered sensor-frame points (xyz, 3 floats each, arrival order;
 * host memory, or device memory when on_device != 0) -> LOAM_B200_C_REG_FULL holds the ring-ordered cloud
 * (x <- y, y <- z, z <- x, intensity = ring + relTime), ring_sizes[n_rings] the points per ring; rejected points
 * (non-finite, |p|^2 < 1e-4, ring outside [0, n_rings)) are dropped.  Follow with loam_b200_reg_run. */
int loam_b200_reg_bin(loam_b200_ctx* ctx, const float* xyz, int n, int on_device, float lower_bound_deg,
                      float upper_bound_deg, int n_rings, float scan_period, int32_t* ring_sizes, int* n_kept);

/* Scan registration on the cloud in LOAM_B200_C_REG_FULL (already uploaded): fills the REG_SHARP / LESS_SHARP / FLAT /
 * LESS_FLAT slots; counts_out[4] = their sizes.  Index lists and labels of this sweep stay readable until the next run. */
int loam_b200_reg_run(loam_b200_ctx* ctx, const int32_t* ring_start, const int32_t* ring_end, int n_rings,
                      const loam_b200_reg_params* params, int counts_out[4]);
/* which: 1 sharp, 2 less sharp, 3 flat */
int loam_b200_reg_indices(loam_b200_ctx* ctx, int which, int32_t* out, int cap, int* n_out);
int loam_b200_reg_labels(loam_b200_ctx* ctx, int8_t* out, int n);

/* Odometry stage on the ODOM_* slots: prepare = take ODOM_SHARP + ODOM_FLAT as this sweep's queries;
 * rebuild_last = BVHs + ring-offset tables over ODOM_LAST_CORNER / ODOM_LAST_SURF (setInputCloud,
 * BasicLaserOdometry.cpp:203-204,662-663), built asynchronously on side streams;
 * loam_b200_odom_iterate (above) then works on them. */
int loam_b200_odom_prepare(loam_b200_ctx* ctx);
/* The registration -> odometry hand-off in one launch: the five clouds of `src_ctx` (src5 = its sharp, less sharp, flat,
 * less flat, full-resolution slots) go to the ODOM_SHARP .. ODOM_FULL slots of `ctx` like loam_b200_cloud_copy_many, and
 * this sweep's query array is filled at the same time (the next loam_b200_odom_prepare then copies nothing). */
int loam_b200_odom_adopt(loam_b200_ctx* ctx, loam_b200_ctx* src_ctx, const int* src5);
int loam_b200_odom_rebuild_last(loam_b200_ctx* ctx);
/* transformToEnd / pointAssociateToMap in place on a device cloud */
int loam_b200_cloud_transform_to_end(loam_b200_ctx* ctx, int slot, const loam_b200_odom_pose* pose);
/* the same on two clouds with one launch (slot_b < 0: only slot_a) */
int loam_b200_cloud_transform_to_end2(loam_b200_ctx* ctx, int slot_a, int slot_b, const loam_b200_odom_pose* pose);
int loam_b200_cloud_transform_to_map(loam_b200_ctx* ctx, int slot, const loam_b200_pose* pose);

/* Mapping stage.  The surrounding map is one point pool per kind (MAP_CORNER_POOL / MAP_SURF_POOL), kept sorted by 1 m
 * cell across sweeps together with its cell table (csrc/mapstore.cuh); the 21x11x21 cube grid of the reference is
 * implicit (a point's cube follows from its position and the grid centre).  Between loam_b200_map_end_sweep and the next
 * loam_b200_map_begin_sweep the host only knows an upper bound of the pool size; loam_b200_cloud_size / _download of
 * the pool slots synchronise and return the exact contents. */
typedef struct {
  int cen[3];                 /* _laserCloudCenWidth / Height / Depth after rolling (BasicLaserMapping.cpp:311-441) */
  const int32_t* valid_cubes; /* _laserCloudValidInd, cube index i + 21 j + 231 k (BasicLaserMapping.h:126-127) */
  int n_valid;                /* <= 125 */
  float corner_leaf, surf_leaf; /* VoxelGrid leaf sizes of the per-cube filters (BasicLaserMapping.cpp:98-99); >= 0.2 m, smaller
                                 * leaves are refused with LOAM_B200_ERR_ARG (8-bit per-axis voxel index inside a cube) */
} loam_b200_map_window;

/* append points (map frame) to the pool of kind 0 corner / 1 surface (unfiltered until their cube is in view at the end
 * of a sweep, like points the reference holds in a cube cloud; the pool is re-sorted at the next begin_sweep) */
int loam_b200_map_pool_append(loam_b200_ctx* ctx, int kind, const float* pts, int n);
/* stacks: MAP_CORNER_LAST / MAP_SURF_LAST -> to map -> back to sensor (predicted pose) -> VoxelGrid -> *_STACK_DS;
 * the field-of-view cube table is uploaded (the search structure itself persists from the previous sweep); queries set
 * for loam_b200_map_iterate / loam_b200_map_solve.
 * sizes_out[4] = number of map points in the valid cubes (corner, surface: the sizes of the reference's
 * laserCloudCornerFromMap / laserCloudSurfFromMap, BasicLaserMapping.cpp:503-509,628), corner_stack_ds, surf_stack_ds */
int loam_b200_map_begin_sweep(loam_b200_ctx* ctx, const loam_b200_pose* predicted, const loam_b200_map_window* win,
                              int sizes_out[4]);
/* insert the stack points with the optimised pose, voxel-filter every valid cube (BasicLaserMapping.cpp:536-593) and
 * move MAP_FULL into the map frame (:595) */
int loam_b200_map_end_sweep(loam_b200_ctx* ctx, const loam_b200_pose* optimised);
/* Same, but issued by a helper thread of the context: returns at once; the next call on this context (any entry point)
 * first waits for the update to be issued and returns its status if it failed. */
int loam_b200_map_end_sweep_async(loam_b200_ctx* ctx, const loam_b200_pose* optimised);
/* createDownsizedMap (:242-264): VoxelGrid(leaf) over the corner + surface points of the surround cubes -> MAP_SURROUND_DS */
int loam_b200_map_surround(loam_b200_ctx* ctx, const int cen[3], const int32_t* surround_cubes, int n, float leaf);
/* Same on an auxiliary context with its own stream and helper thread: returns at once, ordered behind the pending
 * end-of-sweep update; loam_b200_cloud_size / _download of MAP_SURROUND_DS wait for it. */
int loam_b200_map_surround_async(loam_b200_ctx* ctx, const int cen[3], const int32_t* surround_cubes, int n, float leaf);
/* Debug / test switch: loam_b200_map_begin_sweep additionally materialises the reference's laserCloud*FromMap
 * (BasicLaserMapping.cpp:503-509: the map points of the cubes in view) in the *_FROM_MAP cloud slots.  Off by default:
 * the persistent cell-sorted map never needs that copy, only its size (sizes_out[0..1]). */
int loam_b200_map_debug_from_map(loam_b200_ctx* ctx, int on);
/* Test switch: cell pruning of the scan-to-map search over the persistent map (cells a query cannot reach within 1 m are
 * not probed).  mode -1 (default): on when the map's points take more than half of the device's L2; 0 off; 1 on.  The
 * search result does not depend on it. */
int loam_b200_debug_map_prune(loam_b200_ctx* ctx, int mode);
/* Test switch: the scan-to-scan correspondence search scans a ring-ordered last cloud (ring ids 0..255 in ascending order)
 * as two index ranges from its ring offset table.  mode 1 (default): automatic; 0: always the serial scan with the ring
 * `break` (the path every other cloud takes).  Reaches loam_b200_odom_iterate* and loam_b200_odom_solve; the search result
 * does not depend on it. */
int loam_b200_debug_odom_ring_ranges(loam_b200_ctx* ctx, int mode);
/* Test query: how the last build of tree `slot` ran (joins a pending loam_b200_odom_rebuild_last first). */
enum { LOAM_B200_BUILD_NONE = 0, LOAM_B200_BUILD_CLUSTER_PAIR = 1, LOAM_B200_BUILD_CLUSTER = 2,
       LOAM_B200_BUILD_MULTI_LAUNCH = 3 };
int loam_b200_debug_tree_build_path(loam_b200_ctx* ctx, int slot);

/* ------------------------------------------------------------------------------------------------------------------
 * Whole-run voxel map (optional, off by default; csrc/densemap.cuh, DESIGN.md "Whole-run voxel map").  Once enabled,
 * every loam_b200_map_end_sweep(_async) adds the registered full-resolution cloud (MAP_FULL, map frame) to a persistent
 * device hash table of voxels that is never rolled or pruned.  Voxel of a point: (int)floorf(c * (1.0f / leaf)) per
 * axis (PCL VoxelGrid's index before min_b); voxels beyond [-2^20, 2^20) on an axis and non-finite points are skipped.
 * Per voxel: count and fp64 sums, added sequentially in ascending cloud index within a sweep and sweep by sweep; export
 * gives (float)(sum / count) of x, y, z and intensity in ascending voxel order (z-major, x fastest: VoxelGrid's order).
 * When a sweep brings more new voxels than max_voxels leaves room for, they are admitted in ascending voxel order until
 * the table is full and the points of the others are counted as dropped.  The insertion of the mapping stage runs on a
 * stream of its own beside the map update; the next write into MAP_FULL (loam_b200_cloud_upload / _copy / _copy_many /
 * _swap / the in-place transforms, which the drop-in's adopt / laserCloud() / process use) waits for it.
 *   enable: leaf finite and > 0, 1 <= max_voxels <= 2^31 - 1 (else LOAM_B200_ERR_ARG); another leaf while the map holds
 *           voxels, or a sharded context (loam_b200_map_set_shard / comm / peer), gives LOAM_B200_ERR_STATE.  The same
 *           leaf again changes the cap; a cap below the stored voxels keeps them (and their accumulation) and admits
 *           no new voxel.
 *   insert: accumulate the cloud in any slot (kernel-level use and tests; the mapping stage inserts MAP_FULL itself);
 *           everything enqueued on the context afterwards waits for it, since stage calls write some slots directly.
 *   stats:  out3 = voxels, skipped points, dropped points (synchronises).
 *   export: every voxel as packed float[4] centroids (+ counts when counts != NULL); *n_out = number of voxels,
 *           LOAM_B200_ERR_CAPACITY when it exceeds cap (synchronises).  Not enabled: an empty map.
 *   clear:  empty the map (the leaf may then change).
 * Every voxel also keeps two 16-bit evidence counters that saturate at 65535: hits (inserts that put points into it;
 * counted always) and misses (sweeps of the optional visibility pass that saw through it).  They never change the
 * export above.  The visibility pass (off by default; DESIGN.md "Visibility pass") removes moving-object trails:
 *   visibility: h_res_deg, v_res_deg (range-image pixel size) and margin (metres).  Each mapped sweep k, before its
 *           insertion and on the map's stream: with the optimised pose, every finite point of MAP_FULL and every stored
 *           voxel centroid (fp64 sum / count) go to the sensor frame in double (pointAssociateTobeMapped,
 *           BasicLaserMapping.cpp:223-231, with double cos / sin of the negated float angles): range
 *           r = sqrt((x*x + y*y) + z*z), elevation atan2(y, sqrt(x*x + z*z)), azimuth atan2(x, z);
 *           row = clamp(floor((deg(elevation) + 90) / v_res), 0, rows - 1), rows = ceil(180 / v_res);
 *           col = floor((deg(azimuth) + 180) / h_res) mod cols (non-negative), cols = ceil(360 / h_res).  Each pixel
 *           holds the minimum (float) r of the sweep's points with r > 0; a stored voxel whose pixel holds a finite
 *           value v with (double) v > r + margin gets one miss.  Pixels without a return are no evidence.  Cost: one
 *           pass over every table slot per mapped sweep.  h_res_deg == 0 turns it off; non-finite values, h_res
 *           outside (0, 360], v_res outside (0, 180], margin < 0 or rows * cols > 2^24 give LOAM_B200_ERR_ARG; without
 *           the map (or on a sharded context) LOAM_B200_ERR_STATE.
 *   observe: the pass over the cloud in any slot (map frame) seen from `pose` (kernel-level use and tests; the mapping
 *           stage observes MAP_FULL itself); everything enqueued on the context afterwards waits for it.
 *           LOAM_B200_ERR_STATE while the pass is off (in both modes).  It runs whichever mode is on.
 *   carving: the pass's other mode, carve mode (DESIGN.md "Carve mode"), instead of the range image: each mapped sweep,
 *           at the same place, walks every point's ray from the pose's float position o through the map, fp64 without
 *           FMA: e = p - o per axis, r = sqrt((ex*ex + ey*ey) + ez*ez), d = e / r (a non-finite p or r == 0, or an
 *           origin whose voxel lies outside the key range, casts nothing); the walk of loam_b200_dense_raycast from o
 *           along d (start voxel floor(o_a / leaf), ties x, y, z); T = min(r - margin, max_range); the walk ends at the
 *           first voxel with t_exit > T, and each voxel before it that is stored (before the sweep's insertion) is
 *           carved.  K = the voxels of the sweep's own points by the map's rule.  Every stored voxel carved by at least
 *           one ray and not in K gets one miss per sweep (hits win within a sweep), independent of thread order and of
 *           how many rays crossed it.  Cost: O(rays x voxels walked), independent of the map's size; an occupancy
 *           index of 8^3 bricks kept current by the insertion replaces any pass over the table.  max_range == 0 turns
 *           it off.  LOAM_B200_ERR_ARG unless margin >= 0 and max_range >= 0 are finite and max_range / leaf <= 65536.
 *           Without the map (or on a sharded context) LOAM_B200_ERR_STATE.  The two modes exclude each other: turning
 *           one on while the other is on gives LOAM_B200_ERR_STATE.  Misses saturate and feed the exports as above.
 *   export_filtered: the voxels with (double) misses <= max_miss_ratio * (double) hits (max_miss_ratio >= 0; +inf
 *           keeps every voxel and equals loam_b200_dense_export), in ascending voxel order, with the same centroids;
 *           counts, hits and misses may each be NULL.  *n_out = number of voxels kept, LOAM_B200_ERR_CAPACITY when it
 *           exceeds cap (synchronises).
 *   export_normals: the export of export_filtered at max_miss_ratio (same voxels, order, centroids and counts, bit for
 *           bit) plus a surface normal and curvature per voxel, computed over the exported voxels only (a voxel that
 *           the filter removes gets no normal and is nobody's neighbour).  normals: float[4] (nx, ny, nz, curvature)
 *           per voxel, in the centroids' order.  For voxel v with fp32 centroid c_v:
 *             neighbours w: the exported voxels whose index differs from v's by at most `radius` (1..3) on every axis,
 *               v included; an offset outside the key range [-2^20, 2^20) on an axis does not exist (never wraps into
 *               the next row or plane of the key).  Visited in ascending key order (dz, then dy, then dx ascending).
 *             fp64, no FMA, each operation rounded on its own: d = (double)c_w - (double)c_v per axis; S1 += d (3
 *               components); S2 += d_a * d_b (xx, xy, xz, yy, yz, zz); k = number of neighbours;
 *               C_ab = (float)((S2_ab - (S1_a * S1_b) / k) / k).
 *             sym_eigen<3> of C (csrc/linalg.cuh, the 3x3 solver of the scan-to-map line fit): normal = eigenvector of
 *               the smallest eigenvalue; curvature = ev0 / ((ev0 + ev1) + ev2) in fp32, 0 when that sum is 0.
 *             orientation (pcl::flipNormalTowardsViewpoint): with p = viewpoint (map frame, double), the normal is
 *               negated when ((p_x - c_x) * n_x + (p_y - c_y) * n_y) + (p_z - c_z) * n_z < 0 in double.
 *             k < 3, or an eigen-decomposition that does not converge: NaN normal and curvature.
 *           The result is pcl::NormalEstimation's on the exported cloud with a box neighbourhood, each neighbour's
 *           centroid counted once (counts are no weights).  counts may be NULL; xyzi and normals may not once
 *           voxels are exported.  *n_out and LOAM_B200_ERR_CAPACITY as export_filtered; LOAM_B200_ERR_ARG for radius
 *           outside 1..3, a NaN or negative ratio, a NULL or non-finite viewpoint.  Runs only at export, never on the
 *           per-sweep path.
 * ------------------------------------------------------------------------------------------------------------------ */
int loam_b200_dense_enable(loam_b200_ctx* ctx, float leaf, long long max_voxels);
int loam_b200_dense_insert(loam_b200_ctx* ctx, int slot);
int loam_b200_dense_stats(loam_b200_ctx* ctx, long long out3[3]);
int loam_b200_dense_export(loam_b200_ctx* ctx, float* xyzi, uint32_t* counts, int cap, int* n_out);
int loam_b200_dense_clear(loam_b200_ctx* ctx);
int loam_b200_dense_visibility(loam_b200_ctx* ctx, double h_res_deg, double v_res_deg, double margin);
int loam_b200_dense_observe(loam_b200_ctx* ctx, int slot, const loam_b200_pose* pose);
int loam_b200_dense_carving(loam_b200_ctx* ctx, double margin, double max_range);
int loam_b200_dense_export_filtered(loam_b200_ctx* ctx, double max_miss_ratio, float* xyzi, uint32_t* counts,
                                    uint16_t* hits, uint16_t* misses, int cap, int* n_out);
int loam_b200_dense_export_normals(loam_b200_ctx* ctx, double max_miss_ratio, int radius, const double viewpoint[3],
                                   float* xyzi, uint32_t* counts, float* normals, int cap, int* n_out);
/* Test query: slots of the map's hash table as the host sized it last (0 while the map is off).  The table keeps a
 * load factor <= 0.5 of an upper bound of the voxels, so it follows the voxels stored, not the points inserted. */
int loam_b200_debug_dense_table_slots(loam_b200_ctx* ctx, long long* out);
/* Test query: carve mode's occupancy index as rows of 9 words (brick key (v >> 3 per axis of v + 2^20: z << 36 |
 * y << 18 | x), then the 512-bit mask of its voxels, bit (z & 7) << 6 | (y & 7) << 3 | (x & 7)) in ascending brick key;
 * *n_out = its bricks, LOAM_B200_ERR_CAPACITY when they exceed cap rows.  0 bricks while there is no index. */
int loam_b200_debug_dense_carve_index(loam_b200_ctx* ctx, uint64_t* rows, long long cap, long long* n_out);

/* ------------------------------------------------------------------------------------------------------------------
 * Whole-run voxel map snapshots and merging (csrc/densemap.cuh, DESIGN.md "Snapshots and merging"): the accumulator's
 * own state, saved exactly and added back into a map -- resume a stopped run, extend one session's map with another's
 * under the rigid transform dense_relocalize(_global) found, or make a coarser copy.  Not on the per-sweep path.
 *   snapshot: every stored voxel in ascending key order with the fields of its table entry: key (the key codec of
 *           DESIGN.md §5.1: (v_z + 2^20) << 42 | (v_y + 2^20) << 21 | (v_x + 2^20)), count, hits, misses and the four
 *           fp64 sums (x, y, z, intensity) as sums[4 i .. 4 i + 3].  keys, hits and misses may be NULL; counts and sums
 *           may not once voxels are returned (LOAM_B200_ERR_ARG).  *n_out = number of voxels, LOAM_B200_ERR_CAPACITY
 *           when it exceeds cap; not enabled: an empty map.  Synchronous, after everything enqueued on the map's
 *           stream.  (float)(sums / count) equals loam_b200_dense_export's centroids bit for bit; counts, hits and
 *           misses equal loam_b200_dense_export_filtered(+inf)'s.
 *   merge:  add n entries (counts, hits, misses, sums as the snapshot returns them; no keys, no leaf) into the map,
 *           optionally under `pose` (NULL: as stored).  fp64 without FMA, each operation rounded on its own:
 *             S' = S when pose is NULL; otherwise (Sx, Sy, Sz) rotated by rotZ, then rotX, then rotY (as
 *               loam_b200_dense_raycast, with std::cos / std::sin in double of the pose's float angles) and
 *               (double)count * (double)pos_a added per axis; the intensity sum is unchanged.
 *             destination voxel: c_a = (float)(S'_a / (double)count), the key of the map's rule (floorf(c_a * (1.0f /
 *               leaf)) in fp32, the map's current leaf).  So an entry's voxel follows from its centroid: a snapshot
 *               merges into a map of another leaf (into a larger leaf: a coarse copy).  A centroid that is not finite
 *               or whose voxel lies outside the key range is skipped; its count is added to `skipped`.
 *             entries with one destination are combined in ascending input index: P = ((0.0 + S'_i1) + S'_i2) + ...;
 *               counts add (uint32); hits and misses each add with saturation at 65535.
 *             a stored voxel gets S + P, count + the group's count and the saturating sums of its hits and misses; a
 *               new voxel is admitted in ascending key order while the map is under max_voxels (as the insertion
 *               admits one; the count of a group refused is added to `dropped`) with P, the group's count and evidence.
 *               A merge adds no hit of its own: the evidence carried in is the evidence.
 *           Counts add in uint32 as the insertion's do; neither guards against overflow.  With carve mode on, the
 *           voxels admitted enter its occupancy index.  Runs on the map's stream after everything enqueued on the
 *           context; everything enqueued on the context afterwards waits for it.  A target, its ray index, distance
 *           field and place database built earlier do not change.
 *           Every check runs before anything is uploaded, so a refused call changes nothing: LOAM_B200_ERR_ARG for
 *           n < 0, a NULL array with n > 0, an entry with count 0 or hits 0 (every stored voxel has a hit), a sum that
 *           is not finite, or a pose with a non-finite angle or position; LOAM_B200_ERR_STATE without the map or on a
 *           sharded context.  n == 0 launches nothing.
 *   Resume: a snapshot merged into an empty map of the same leaf with pose NULL reproduces it bit for bit -- each
 *   entry lands in its own voxel (a centroid lies between its points and floorf is monotone), and 0.0 + S == S since
 *   a stored sum is never -0.0 -- so inserting the remaining sweeps afterwards gives the map of a run that never
 *   stopped.  A zero pose gives the same bits as NULL on snapshot input.  Launches count under LOAM_B200_K_DENSE.
 * ------------------------------------------------------------------------------------------------------------------ */
int loam_b200_dense_snapshot(loam_b200_ctx* ctx, uint64_t* keys, uint32_t* counts, uint16_t* hits, uint16_t* misses,
                             double* sums, int cap, int* n_out);
int loam_b200_dense_merge(loam_b200_ctx* ctx, const uint32_t* counts, const uint16_t* hits, const uint16_t* misses,
                          const double* sums, int n, const loam_b200_pose* pose);

/* ------------------------------------------------------------------------------------------------------------------
 * Alignment against the whole-run voxel map (csrc/densemap.cuh, DESIGN.md "Alignment against the whole-run voxel map"):
 * point-to-plane Gauss-Newton of a cloud against a device-resident target of voxel centroids and normals, for
 * relocalisation in a map built earlier, drift checks of a mapped pose, or placing another sensor's or session's sweeps
 * in the same map.  Not on the per-sweep path; the result never feeds back into the mapping stage.
 *   target_build: the target is the export of loam_b200_dense_export_normals(max_miss_ratio, radius, viewpoint) --
 *           the same voxels, order and bits -- kept on the device as sorted keys, centroids and normals.  A snapshot:
 *           later inserts do not change it; the next build or load replaces it; destroying the context frees it.
 *           *n_out = its voxels.  Arguments as export_normals (LOAM_B200_ERR_ARG); without the map, or on a sharded
 *           context, LOAM_B200_ERR_STATE.
 *   target_load: the target from n host entries (a map saved earlier): xyzi float[4] centroids, normals float[4]
 *           (nx, ny, nz, anything: the export_normals layout); a NaN nx means "no normal".  Works with or without the
 *           map.  An entry's voxel is dense_key_of(centroid, 1.0f / leaf) (the map's voxel rule); entries are sorted
 *           by it.  LOAM_B200_ERR_ARG for a leaf that is not finite and > 0, a centroid that is not finite or whose
 *           voxel is outside the key range, or two entries in one voxel.  Export -> load gives back the built target
 *           exactly: a centroid (float)(S / count) lies between the smallest and largest of its voxel's points and
 *           floorf(c * inv) is monotone in c, so an exported centroid's voxel is its own voxel.
 *   A failed build or load leaves no target.
 *   align_iterate: one iteration over n points (sensor frame, float[4]; host memory, or device memory when
 *           on_device != 0) at `pose`, fp32 without FMA, each operation rounded on its own:
 *             q = pointAssociateToMap(pose, p) with the pose's sin / cos (as loam_b200_map_iterate); a non-finite p
 *               has no correspondence; v = q's voxel (the target's leaf); v outside the key range: none.
 *             candidates: the target voxels within search_radius (1..3) of v on every axis with a normal, in ascending
 *               key order (an offset outside the key range does not exist); d = c - q, d2 = (dx*dx + dy*dy) + dz*dz;
 *               the first smallest d2 wins and is accepted when d2 < gate, gate = s * s with s = (float)search_radius *
 *               leaf, both rounded to fp32.  The box contains the ball of radius s around q, so an accepted match is
 *               the exact nearest centroid with a normal within that distance.
 *             pd2 = (nx*(qx - cx) + ny*(qy - cy)) + nz*(qz - cz); s = 1 - 0.9f * |pd2| / sqrtf(sqrtf((px*px + py*py)
 *               + pz*pz)) with the SENSOR-frame p; selected when (double)s > 0.1; coeff = (s*nx, s*ny, s*nz, s*pd2).
 *             Jacobian row and rhs = -coeff.w of loam_b200_map_iterate.
 *           ne: the normal equations over the selected rows; n_selected; n_corner_selected = 0.  sum_pd2_sq: the fp32
 *           sum of pd2^2 over the selected rows.  Sums: per warp of 32 points an fp32 xor butterfly, per CTA of 128
 *           points the 4 warp sums in warp order, then the CTA partials in double (warp w of the last CTA folds CTAs
 *           w, w + 4, ...; the 4 results added in warp order), rounded to fp32 once -- run-to-run deterministic.
 *           Per point (each may be NULL): dbg_match = target index (ascending key order) of the accepted match or -1,
 *           dbg_coeff = coeff (float[4]; 0 without a match), dbg_sel = 1 when selected.
 *   align: Gauss-Newton from `initial` with the mapping stage's policy (BasicLaserMapping.cpp:826-922): an iteration
 *           with fewer than 50 selected rows is skipped; 6x6 solve with eigenvalue threshold 100, the degeneracy
 *           projection computed on the first iteration that reaches the solve and kept; float pose update, sin / cos
 *           recomputed from the float angles (loam::Angle); stop when deltaR < 0.05 deg and deltaT < 0.05 cm, or after
 *           max_iterations (1..100).  One kernel launch and a 32-float readback per iteration.  An empty cloud or an
 *           empty target runs nothing: the pose comes back unchanged with iterations = 0.  Coarse to fine: call twice
 *           (search_radius 3, then 1 from the first result).
 *   No target: LOAM_B200_ERR_STATE.  A bad radius or iteration count, a NULL pointer or a non-finite pose (rot, sin,
 *   cos or pos): LOAM_B200_ERR_ARG.  Launches count under LOAM_B200_K_DENSE.
 * ------------------------------------------------------------------------------------------------------------------ */
typedef struct {
  float rot[3];    /* aligned rot_x, rot_y, rot_z */
  float pos[3];
  int iterations;  /* iterations executed (0: nothing to align) */
  int n_selected;  /* selected rows of the last executed iteration, at that iteration's input pose */
  float rms;       /* sqrt(sum pd2^2 / n_selected) of that iteration (double, rounded once; 0 when none selected) */
  int degenerate;  /* the solve's degeneracy projection is in effect */
  int converged;   /* stopped by the deltaR / deltaT thresholds, not by max_iterations */
} loam_b200_align_result;

int loam_b200_dense_target_build(loam_b200_ctx* ctx, double max_miss_ratio, int radius, const double viewpoint[3],
                                 int* n_out);
int loam_b200_dense_target_load(loam_b200_ctx* ctx, float leaf, const float* xyzi, const float* normals, int n);
int loam_b200_dense_align_iterate(loam_b200_ctx* ctx, const float* xyzi, int n, int on_device,
                                  const loam_b200_pose* pose, int search_radius, loam_b200_normal_eq* ne,
                                  float* sum_pd2_sq, int32_t* dbg_match, float* dbg_coeff, int8_t* dbg_sel);
int loam_b200_dense_align(loam_b200_ctx* ctx, const float* xyzi, int n, int on_device, const loam_b200_pose* initial,
                          int search_radius, int max_iterations, loam_b200_align_result* out);

/* ------------------------------------------------------------------------------------------------------------------
 * Relocalisation against the whole-run voxel map (DESIGN.md "Relocalisation against the whole-run voxel map"): one
 * cloud at many poses against the target above, for a restart or a tracking loss where the position is roughly known
 * (the last saved pose, GNSS) and the heading is not.  Not on the per-sweep path; the result never feeds back into
 * the mapping stage.  The target, cloud, radius, iteration and error rules are those of align_iterate / align.
 *   dense_score: the k poses (1 <= k <= 1 << 20) in one upload of the cloud and one launch per chunk of at most
 *           65535 poses -> per pose exactly what align_iterate returns at that pose in ne.n_selected and sum_pd2_sq.
 *   dense_align_batch: k independent runs of align from initial[h] -> out[h], equal to dense_align from initial[h]
 *           bit for bit (the same host solve and degeneracy projection per run).  Per iteration one launch per chunk
 *           over the runs still going and one readback; a run leaves when it converges or after max_iterations.
 *           dense_align is this with k = 1.
 *   reloc_grid: host only.  The LOAM frame has y up: heading is rot_y, the ground plane x-z.  The poses, j outer,
 *           then iz, then ix, each ascending from -steps to +steps:
 *             rot_y = prior.rot_y + (float)((double)j * yaw_step_deg * pi / 180), rot_x / rot_z the prior's,
 *             pos = (prior.x + (float)ix * xz_step, prior.y, prior.z + (float)iz * xz_step), all in float;
 *             sin_ / cos_ = std::sin / std::cos of the float angles (loam::Angle).
 *           (2 yaw_steps + 1) (2 xz_steps + 1)^2 poses, at most 1 << 20; a full circle is yaw_steps =
 *           ceil(180 / yaw_step_deg) (the duplicated +-180 deg is harmless).  *n_out = that count;
 *           LOAM_B200_ERR_CAPACITY when it exceeds cap.  LOAM_B200_ERR_ARG for a step that is not finite and > 0, a
 *           negative step count, a non-finite prior or a NULL pointer.
 *   dense_relocalize: built on the two calls above, in this order:
 *           1. score every hypothesis at score_radius;
 *           2. keep the `keep` best (1..1024) by selected descending, then index ascending; one with fewer than 50
 *              selected is never kept (it could not take a step);
 *           3. dense_align_batch of the kept poses at coarse_radius, then at fine_radius from those results (sin /
 *              cos recomputed from the float angles), each with max_iterations;
 *           4. score at fine_radius at the refined poses -> selected, rms = sqrt(sum pd2^2 / selected) in double,
 *              rounded once (0 when none);
 *           5. rank by selected descending, then rms ascending, then keep order;
 *           6. drop a candidate whose translation differs from a better-ranked survivor's by less than dedup_m AND
 *              whose rotation differs by less than dedup_deg (the angle of R(a)^T R(b), in double);
 *           7. write the first cap survivors; *n_out = candidates written (0, with no error, when nothing reaches 50).
 *           The gap between candidates 0 and 1 is the ambiguity of the result.  A host cloud is uploaded once.
 *   Errors: no target LOAM_B200_ERR_STATE; a bad radius, iteration count, keep, k, cap or dedup threshold (negative
 *   or not finite), a NULL pointer or a non-finite pose LOAM_B200_ERR_ARG.  An empty cloud or target runs nothing:
 *   scores are 0, every run returns its initial pose with iterations = 0, relocalize returns no candidate.
 *   Launches count under LOAM_B200_K_DENSE.
 * ------------------------------------------------------------------------------------------------------------------ */
typedef struct {
  int score_radius;   /* search radius of the first score (1..3) */
  int coarse_radius;  /* of the first refinement */
  int fine_radius;    /* of the second refinement and the final score */
  int keep;           /* hypotheses refined (1..1024) */
  int max_iterations; /* per refinement (1..100) */
  float dedup_m;      /* duplicate: closer than this in translation (>= 0) ... */
  float dedup_deg;    /* ... and than this in rotation (>= 0) */
} loam_b200_reloc_params;

typedef struct {
  int hypothesis;                /* index into the hypotheses given */
  int score_selected;            /* its selected count in the first score */
  loam_b200_align_result coarse; /* the refinement at coarse_radius */
  loam_b200_align_result fine;   /* the refinement at fine_radius from the coarse pose: the candidate's pose */
  int selected;                  /* the final score at the fine pose */
  float rms;
} loam_b200_reloc_candidate;

/* Recommended parameters, chosen from the measured basin (DESIGN.md "Relocalisation against the whole-run voxel
 * map"): a full-circle yaw grid at 2 deg (90 steps to each side) and an x-z grid of 0.4 m steps four to each side of
 * the prior (+-1.6 m), 181 x 81 = 14661 poses.  The nearest grid pose is then within 1 deg and 0.2 m per axis (0.28 m)
 * of the truth, a corner from which every measured coarse-to-fine run converged (VLP-16 and HDL-64E, leaf 0.1 and 0.2,
 * 8 directions, both yaw signs). */
#define LOAM_B200_RELOC_YAW_STEP_DEG 2.0f
#define LOAM_B200_RELOC_XZ_STEP 0.4f
#define LOAM_B200_RELOC_XZ_STEPS 4
#define LOAM_B200_RELOC_PARAMS_DEFAULT {3, 3, 1, 16, 30, 0.5f, 5.0f}

int loam_b200_dense_score(loam_b200_ctx* ctx, const float* xyzi, int n, int on_device, const loam_b200_pose* poses,
                          int k, int search_radius, int32_t* n_selected, float* sum_pd2_sq);
int loam_b200_dense_align_batch(loam_b200_ctx* ctx, const float* xyzi, int n, int on_device,
                                const loam_b200_pose* initial, int k, int search_radius, int max_iterations,
                                loam_b200_align_result* out);
int loam_b200_reloc_grid(const loam_b200_pose* prior, float yaw_step_deg, int yaw_steps, float xz_step, int xz_steps,
                         loam_b200_pose* out, int cap, int* n_out);
int loam_b200_dense_relocalize(loam_b200_ctx* ctx, const float* xyzi, int n, int on_device,
                               const loam_b200_pose* hyps, int k, const loam_b200_reloc_params* prm,
                               loam_b200_reloc_candidate* out, int cap, int* n_out);

/* ------------------------------------------------------------------------------------------------------------------
 * Ray casting the whole-run voxel map (csrc/densemap.cuh, DESIGN.md "Ray casting the whole-run voxel map"): what the
 * sensor should see from a pose in the target above -- change detection between sessions, a check of a pose found by
 * dense_align / dense_relocalize, simulated scans.  Not on the per-sweep path; the result never feeds back into the
 * mapping stage.  n rays (float[4] in the sensor frame, w ignored: a sweep's own points may be passed; host memory,
 * or device memory when on_device != 0) from `pose`, fp64 without FMA, each operation rounded on its own, no
 * transcendental function on the device:
 *   ray: |p| = sqrt((x*x + y*y) + z*z) in double of the float components, u = p / |p|; d = u rotated into the map frame
 *     by rotZ, then rotX, then rotY (associate_to_map's order) with std::cos / std::sin in double of the pose's float
 *     angles; origin o = the pose's float pos as double.  A non-finite or zero p has no hit.
 *   voxels: L = (double)leaf of the target; voxel v spans [v L, (v + 1) L) per axis; the start voxel is floor(o_a / L);
 *     a voxel is occupied when its key is in the target (indices outside [-2^20, 2^20) never are).
 *   walk (Amanatides-Woo with exact re-evaluation): per axis with d_a != 0, inv_a = 1.0 / d_a and t_next_a =
 *     ((double)k L - o_a) inv_a, k = v_a + 1 when d_a > 0, v_a when d_a < 0; +inf when d_a == 0.  The voxel spans
 *     [t_enter, t_exit = min t_next), the first one from t_enter = 0.  A step goes along the axis of the smallest t_next
 *     (ties: x, then y, then z); the next voxel's t_enter is that axis's old t_next, and only its t_next is recomputed,
 *     from the new index.
 *   hit: the first occupied voxel with t_exit > min_range; lo = max(t_enter, min_range), hi = t_exit.  With a normal
 *     (nx not NaN): den = (nx dx + ny dy) + nz dz, num = (nx (cx - ox) + ny (cy - oy)) + nz (cz - oz) with the float
 *     centroid and normal as double, and t = clamp(num / den, lo, hi) when den != 0; otherwise t = lo.  The surfel
 *     gives a sub-voxel range on surfaces; the first occupied voxel always stops the ray, so there are no holes.
 *   out: the walk ends with no hit when t_enter > max_range or the hit's t > max_range.  A hit: range[i] = (float)t,
 *     index[i] = the voxel's position in the target's ascending key order (the export's order for a built target).
 *     No hit: range[i] = +inf, index[i] = -1.  index may be NULL.  Synchronous.
 * A ray index (a hash table of 8^3-voxel bricks with a 512-bit occupancy mask each) is built on the first cast after a
 * target build or load and kept with the target.  No target: LOAM_B200_ERR_STATE.  LOAM_B200_ERR_ARG unless
 * 0 <= min_range < max_range (both finite), max_range / leaf <= 65536 (every walk is then at most ~3 * 2^16 steps),
 * the pose is finite and its position's voxel lies in the key range; and for a NULL pointer.  An empty target or
 * n = 0 returns no hits and launches nothing.  Launches count under LOAM_B200_K_DENSE.
 * ------------------------------------------------------------------------------------------------------------------ */
int loam_b200_dense_raycast(loam_b200_ctx* ctx, const float* rays, int n, int on_device, const loam_b200_pose* pose,
                            float min_range, float max_range, float* range, int32_t* index);
/* Test query: device bytes of the target's ray index (0 until the first cast after a build or load). */
int loam_b200_debug_dense_ray_index_bytes(loam_b200_ctx* ctx, long long* out);

/* ------------------------------------------------------------------------------------------------------------------
 * Distance field of the whole-run voxel map (csrc/densemap.cuh, DESIGN.md "Distance field of the whole-run voxel
 * map"): how far a point is from the nearest obstacle of the target above, and in which direction that distance grows
 * -- collision checks, safety margins, trajectory optimisers.  Not on the per-sweep path; the field never feeds back
 * into the mapping stage.  Unsigned (0 inside obstacles), no unknown space.
 *   occupied: a voxel whose key is in the target (as for the ray cast: with or without a normal).  L = (double)leaf of
 *     the target; voxel v spans [v L, (v + 1) L) per axis.
 *   box: lo[3] (voxel indices, e.g. floorf(c * (1.0f / leaf)) of a corner, api.voxel_box) and dims[3] >= 1, axis-
 *     aligned in the map frame (the LOAM frame, y up).  Cell (x, y, z) is voxel lo + (x, y, z); x varies fastest,
 *     then y, then z (numpy shape (nz, ny, nx)).
 *   value: sq = the squared Euclidean distance in voxel units from the cell's voxel to the nearest occupied voxel of
 *     the whole target, centre to centre (an integer, 0 on an occupied cell); dist = (float)(sqrt((double)sq) * L).
 *   range: max_distance (finite, > 0).  A cell is beyond when sqrt((double)sq) * L > (double)max_distance; a beyond
 *     cell has sq = -1 and dist = +inf.  The exact transform runs over the box grown by pad = floor((double)
 *     max_distance / L) + 1 voxels on every side: an obstacle within max_distance of a cell lies inside that padded
 *     box, so every value reported equals the whole-target value and every beyond cell is truly beyond.
 * build: dist and sq (nx * ny * nz each) may each be NULL (the field is then kept on the device only).  The field (sq,
 *   4 B per cell) is a snapshot kept with the target: later inserts do not change it, the next build replaces it, a
 *   target build or load drops it.  The first build after a target build or load also builds the target's ray index
 *   (loam_b200_dense_raycast) and rasterises from it; an empty target gives a field beyond everywhere and launches
 *   nothing.  Synchronous.
 * query: n points (float[4] in the map frame, w ignored; host memory, or device memory when on_device != 0) ->
 *   dist[n] and, unless grad is NULL, grad[3n] (d dist / d x, y, z per point).  fp64 without FMA, each operation
 *   rounded on its own, one rounding to float at the end:
 *     per axis a: g_a = ((double)p_a / L - 0.5) - (double)lo_a; defined when dims_a >= 2 and 0 <= g_a <= dims_a - 1 on
 *       every axis (a NaN or infinite coordinate never is): then i_a = min((int)floor(g_a), dims_a - 2), f_a = g_a -
 *       i_a; otherwise dist and grad are NaN.
 *     corner w(dx, dy, dz) = sqrt((double)sq) * L of cell i + (dx, dy, dz), or (double)max_distance for a beyond
 *       corner (the query saturates there); lerp(a, b, f) = a + f * (b - a).
 *     dist = lerp(lerp(lerp(w000, w100, fx), lerp(w010, w110, fx), fy), lerp(lerp(w001, w101, fx), lerp(w011, w111,
 *       fx), fy), fz)   (w indexed x y z)
 *     gx = lerp(lerp(w100 - w000, w110 - w010, fy), lerp(w101 - w001, w111 - w011, fy), fz) / L
 *     gy = lerp(lerp(w010 - w000, w110 - w100, fx), lerp(w011 - w001, w111 - w101, fx), fz) / L
 *     gz = lerp(lerp(w001 - w000, w101 - w100, fx), lerp(w011 - w010, w111 - w110, fx), fy) / L
 * No target, or a query without a field: LOAM_B200_ERR_STATE.  LOAM_B200_ERR_ARG for a NULL pointer (lo, dims; xyzi
 * or dist with n > 0), a non-finite max_distance, unless max_distance > 0, max_distance / leaf <= 1024, every padded
 * axis dims_a + 2 pad <= 8192, the padded cells <= 2^27 and the padded box inside the key range [-2^20, 2^20).
 * Launches count under LOAM_B200_K_DENSE.
 * ------------------------------------------------------------------------------------------------------------------ */
int loam_b200_dense_distance_build(loam_b200_ctx* ctx, const int lo[3], const int dims[3], float max_distance,
                                   float* dist, int32_t* sq);
int loam_b200_dense_distance_query(loam_b200_ctx* ctx, const float* xyzi, int n, int on_device, float* dist,
                                   float* grad);
/* Test query: device bytes of the distance field (4 per cell of the box; 0 without a field). */
int loam_b200_debug_dense_distance_bytes(loam_b200_ctx* ctx, long long* out);

/* ------------------------------------------------------------------------------------------------------------------
 * Place recognition and global relocalisation in the whole-run voxel map (csrc/densemap.cuh, DESIGN.md "Place
 * recognition and global relocalisation"): relocalise a cloud with no prior pose -- a robot waking up in a saved map,
 * a tracking loss after a long gap, a second session that starts elsewhere.  A polar height descriptor of the cloud
 * is compared with descriptors rendered from the target at candidate places, over every heading; the best places,
 * each with a heading, become a small dense_relocalize grid.  Not on the per-sweep path.
 *   Descriptor (rings x sectors cells, ring-major, float), LOAM frame: y is up, the ground plane x-z, heading rot_y.
 *     Per point (float[4] in the sensor frame, w ignored), fp64 without FMA, each operation rounded on its own:
 *       a non-finite point is skipped; r = sqrt(x*x + z*z); skipped when r == 0 or r >= max_radius;
 *       ring = floor(r / w) with w = (double)max_radius / rings on the host, clamped to rings - 1;
 *       sector: the wedge [k D, (k + 1) D), D = (2 pi) / sectors in double, that holds the azimuth atan2(x, z), found
 *         without a transcendental function on the device: the number of boundaries k in [1, sectors) that the point
 *         is at or past, where past(k) = h_p > h_k, or h_p == h_k and x * cos(k D) - z * sin(k D) >= 0; h_k = 1 when
 *         2k >= sectors (else 0), h_p = 0 when x > 0 or (x == 0 and z > 0) (else 1); cos / sin are std::cos /
 *         std::sin in double of (double)k * D on the host, except (-1, 0) exactly for the boundary at pi (2k ==
 *         sectors).  past() then holds on a prefix of the boundaries, so the device bisects;
 *       value v = (float)(y + height_offset); a point with v not in (0, FLT_MAX] is skipped.
 *     A cell holds the largest value of its points, 0 when it has none.  Bit-reproducible in any thread order.
 *     Headings: to_map rotates a sensor-frame azimuth phi to phi + rot_y, so query column j matching database column
 *     (j + s) mod sectors means heading s D, reported wrapped to (-pi, pi]: yaw = (float)((double)a * D) with a = s
 *     when 2s <= sectors, else s - sectors.
 *   place_descriptor: the descriptor of n points (host, or device when on_device != 0) -> out[rings * sectors].
 *   dense_place_build: the place database of the current target: k candidate positions (float[3], map frame) and
 *     n_rays sensor-frame rays (float[4]: lidar_rays with the query sensor's elevations and an azimuth count that is
 *     a multiple of sectors).  Candidate c's descriptor is, by definition, place_descriptor of the points
 *     (float)((double)range_i * u_i) per axis over the rays i that hit, where (range, u) are loam_b200_dense_raycast's
 *     from the pose rot = 0, pos = positions[c] with params.min_range / max_range (u = p / |p| of that call).  Rendering
 *     through the cast keeps occlusion.  The ray index is built first when absent.  The database belongs to the
 *     target: the next target build or load drops it, later inserts do not change it; it is a function of (target,
 *     positions, rays, params), so a loaded target and the saved positions rebuild it exactly.  A build replaces the
 *     previous database.  LOAM_B200_ERR_ARG: 1 <= rings <= 64, 1 <= sectors <= 720, rings * sectors <= 4096, max_radius
 *     finite > 0, height_offset finite, the cast's range rules (0 <= min_range < max_range, finite, max_range / leaf
 *     <= 65536), 1 <= k <= 1 << 20, every position finite with its voxel in the key range, n_rays >= 0, no NULL
 *     pointer.  LOAM_B200_ERR_CAPACITY: k * rings * sectors * 4 bytes above LOAM_B200_PLACE_MAX_BYTES.
 *   dense_place_query: the descriptor of the cloud (as place_descriptor, with the database's params), then every
 *     candidate at every shift s in [0, sectors): per column j ascending, query column j against candidate column
 *     (j + s) mod sectors; qq, dd and dot are fp64 sums in ascending ring; a column with qq == 0 or dd == 0 is
 *     skipped, otherwise sim = dot / (sqrt(qq) * sqrt(dd)) is added; dist = 1 - sum / counted (+inf when none is
 *     counted).  Per candidate the best shift: smallest dist, ties to the smaller s.  out: the top_m (1..1024)
 *     candidates by dist ascending, then index ascending, never one at +inf; *n_out = entries written.  No database:
 *     LOAM_B200_ERR_STATE.
 *   place_grid: host only.  For each match m in order, loam_b200_reloc_grid of the prior (rot = (0, yaw_m, 0), pos =
 *     pos_m) with the given steps, concatenated; *n_out = the total (LOAM_B200_ERR_CAPACITY above cap, LOAM_B200_ERR_ARG
 *     above 1 << 20 or for the grid's argument errors).
 *   dense_relocalize_global: dense_place_query(top_m), then loam_b200_dense_relocalize on the place_grid of its
 *     matches -- bit for bit that call on that list; a host cloud is uploaded once.  A candidate's hypothesis indexes
 *     the list, so its match is hypothesis / ((2 yaw_steps + 1) (2 xz_steps + 1)^2); query + place_grid regenerate the
 *     list.  No match: no candidate.  Errors are those of the three calls.
 *   Launches count under LOAM_B200_K_DENSE.  With none of these called nothing is launched, allocated or recorded.
 * ------------------------------------------------------------------------------------------------------------------ */
typedef struct {
  int rings;           /* N_r, 1..64 */
  int sectors;         /* N_s, 1..720, rings * sectors <= 4096 */
  float max_radius;    /* metres, > 0 */
  float height_offset; /* metres added to y before the value (the sensor's height above the ground, or more) */
  float min_range;     /* the database's cast: loam_b200_dense_raycast's min_range ... */
  float max_range;     /* ... and max_range */
} loam_b200_place_params;

typedef struct {
  int candidate; /* index into the positions of dense_place_build */
  int shift;     /* the best shift s */
  float yaw;     /* its heading s D wrapped to (-pi, pi] */
  float pos[3];  /* the candidate's position */
  double dist;   /* its distance */
} loam_b200_place_match;

/* Recommended parameters, chosen from the recall measured on route maps (DESIGN.md "Place recognition and global
 * relocalisation"): 20 rings, 60 sectors (6 deg), 80 m, height offset 2 m, the database cast from 0 to 100 m; places
 * every 4 m along the route; the global relocalisation refines the 5 best places over +-3 steps of 2 deg and an x-z
 * grid of 0.4 m steps five to each side (+-2 m): 5 x 7 x 121 = 4235 poses. */
#define LOAM_B200_PLACE_PARAMS_DEFAULT {20, 60, 80.0f, 2.0f, 0.0f, 100.0f}
#define LOAM_B200_PLACE_SPACING 4.0f
#define LOAM_B200_PLACE_TOP_M 5
#define LOAM_B200_PLACE_YAW_STEP_DEG 2.0f
#define LOAM_B200_PLACE_YAW_STEPS 3
#define LOAM_B200_PLACE_XZ_STEP 0.4f
#define LOAM_B200_PLACE_XZ_STEPS 5
#define LOAM_B200_PLACE_MAX_BYTES (1ll << 30)

int loam_b200_place_descriptor(loam_b200_ctx* ctx, const float* xyzi, int n, int on_device,
                               const loam_b200_place_params* prm, float* out);
int loam_b200_dense_place_build(loam_b200_ctx* ctx, const float* positions, int k, const float* rays, int n_rays,
                                const loam_b200_place_params* prm);
int loam_b200_dense_place_query(loam_b200_ctx* ctx, const float* xyzi, int n, int on_device, int top_m,
                                loam_b200_place_match* out, int* n_out);
int loam_b200_place_grid(const loam_b200_place_match* matches, int n_matches, float yaw_step_deg, int yaw_steps,
                         float xz_step, int xz_steps, loam_b200_pose* out, int cap, int* n_out);
int loam_b200_dense_relocalize_global(loam_b200_ctx* ctx, const float* xyzi, int n, int on_device, int top_m,
                                      float yaw_step_deg, int yaw_steps, float xz_step, int xz_steps,
                                      const loam_b200_reloc_params* prm, loam_b200_reloc_candidate* out, int cap,
                                      int* n_out);
/* Test query: the database's descriptors, k * rings * sectors floats in candidate order -> out; *n_out = that count
 * (0 without a database), LOAM_B200_ERR_CAPACITY when it exceeds cap. */
int loam_b200_debug_dense_place_descriptors(loam_b200_ctx* ctx, float* out, long long cap, long long* n_out);

/* ------------------------------------------------------------------------------------------------------------------
 * Euclidean segmentation of the whole-run voxel map and of clouds (csrc/densemap.cuh, DESIGN.md "Euclidean
 * segmentation"): which voxels or points belong together -- dropping small specks from an export, grouping the points
 * of a sweep that the map does not explain into objects.  pcl::EuclideanClusterExtraction's semantics, computed exactly.
 * Not on the per-sweep path; neither call changes the map, the target or any product of the target (ray index,
 * distance field, place database).
 *   entries: each has a float position p_i and a key k_i of the map's codec at cell size `cell`.
 *     dense_segment: the target's voxels in ascending key order (dense_raycast's index), p_i = the centroid, k_i = the
 *       target's key, cell = the target's leaf.  A built or a loaded target.
 *     cloud_segment: n points (float[4], w ignored; host memory, or device memory when on_device != 0); k_i =
 *       floorf(c * (1.0f / tol)) per axis as the map keys a point (cell = tol).  A point that is not finite or whose
 *       voxel lies outside [-2^20, 2^20) is not an entry (label -1), as the insertion skips it.
 *   candidates: r = floor((double)tol / (double)cell) + 1; the pairs (i, j) whose voxels lie within r voxels of each
 *     other on every axis (the rows of dense_box_walk: per (z, y) row inside the key range, never wrapping).  Two
 *     points within tol lie at most ceil(tol / cell) <= r cells apart on each axis in exact arithmetic.  The keying is
 *     monotonic, and fp32 keying or a centroid's fp32 rounding moves a point across at most the one face it lies on;
 *     where tol / cell is an integer (always in cloud mode) the +1 leaves the spare cell that absorbs that move, and
 *     elsewhere the pair would have to lie further than tol apart to gain a cell.  Only a tol / cell within a few
 *     fp32 ulps below an integer leaves a pair at the very limit outside; the box at r is the definition.
 *   edge: a candidate pair with d2 <= (double)tol * (double)tol, d2 = (dx*dx + dy*dy) + dz*dz, dx = (double)p_i.x -
 *     (double)p_j.x (likewise y, z), fp64 without FMA, each operation rounded on its own.
 *   segment: a connected component of the edge graph; those with min_size <= size <= max_size are kept.
 *   rank: size descending, ties by the smallest entry index (the position in key order for a target, the input index
 *     for a cloud); ids 0..K-1 in that order.
 *   labels[i]: the entry's segment id, -1 when its segment was filtered out or it is not an entry; in entry order (key
 *     order for a target, input order for a cloud).  May be NULL.
 *   record: size, first = the smallest entry index, lo / hi = the float min / max of the members' coordinates per axis,
 *     centroid = (float)(sum / size) per axis.  The fp64 sums: members in ascending entry index, in consecutive chunks
 *     of 256 from the segment's first member; each chunk summed one member after the other from 0.0 ((double) of the
 *     float coordinate), then the chunk sums added in chunk order from 0.0.
 *   out: segments[0 .. K) and *n_out = K; LOAM_B200_ERR_CAPACITY (with *n_out = K, nothing else written) when K > cap.
 * Union-find with atomic hooks of the larger root under the smaller: every root is the smallest member of its
 * component, so the result does not depend on thread scheduling; every output above is exact and reproducible.
 * LOAM_B200_ERR_ARG: tol not finite or not > 0, tol / leaf > 4 for a target (r <= 5, at most 121 rows per entry; for a
 * coarser tolerance merge a snapshot into a coarser map and build a target from it), min_size < 1, min_size >
 * max_size, n < 0, cap < 0, a NULL pointer (segments with cap > 0, n_out; xyzi with n > 0).  dense_segment without a
 * target: LOAM_B200_ERR_STATE.  Every check runs on the host before anything is launched, so a refused call changes
 * nothing.  An empty target or cloud launches nothing (K = 0).  Synchronous.  Launches count under LOAM_B200_K_DENSE,
 * a fixed number per call for a given entry count (the union-find runs one pass, whatever the data).
 * Cost: the union pass visits, per entry, every entry of its box of (2r + 1)^3 voxels.  A target holds one entry per
 * voxel and r <= 5, so that is at most 1331 visits per entry.  A cloud is keyed at cell = tol, so one voxel holds every
 * point of a tol-sized cube and the pass grows with the square of the points per voxel: O(n^2) when a whole cloud
 * falls into a few voxels (a tolerance of metres on a dense sweep, most of whose points lie near the sensor).  For a
 * large tolerance, thin the cloud first (loam_b200_voxel_grid at a fraction of tol) or segment a target built from it.
 * ------------------------------------------------------------------------------------------------------------------ */
typedef struct {
  int32_t size;        /* members */
  int32_t first;       /* the smallest entry index of its members */
  float lo[3], hi[3];  /* min / max of the members' x, y, z */
  float centroid[3];   /* (float)(fp64 sum / size) per axis */
} loam_b200_segment;

/* the current target's voxels: the length of dense_segment's labels (LOAM_B200_ERR_STATE without a target) */
int loam_b200_dense_target_size(loam_b200_ctx* ctx, int* n_out);
int loam_b200_dense_segment(loam_b200_ctx* ctx, float tol, int min_size, int max_size, int32_t* labels,
                            loam_b200_segment* segments, int cap, int* n_out);
int loam_b200_cloud_segment(loam_b200_ctx* ctx, const float* xyzi, int n, int on_device, float tol, int min_size,
                            int max_size, int32_t* labels, loam_b200_segment* segments, int cap, int* n_out);

/* ------------------------------------------------------------------------------------------------------------------
 * Ground of the whole-run voxel map (csrc/densemap.cuh dense_ground_*, DESIGN.md "Ground patches"): which target
 * voxels are ground, the segmentation of everything else, and which points of a sweep lie on the ground the map
 * knows -- the step before grouping objects.  The map frame is LOAM's, y up: the ground plane is x-z.  Not on the
 * per-sweep path; no call changes the map, the target, its ray index, distance field or place database, or an earlier
 * segmentation's result.  Synchronous.  Launches count under LOAM_B200_K_DENSE.
 * dense_ground (a built or loaded target; params below):
 *   candidate: a target voxel whose normal_x is not NaN and (double)fabsf(n_y) >= cos_max, cos_max = cos(max_slope_deg
 *     * pi / 180) in double (the normal's orientation is irrelevant), and n_w <= max_curvature in fp32 (a NaN w fails)
 *     unless max_curvature is +inf, which skips the curvature test (a loaded target whose w means nothing).
 *   candidate pairs: dense_box_walk at r = floor(max(tol, max_step) / leaf) + 1 over the candidates in key order.
 *   edge: both candidates, dx*dx + dz*dz <= tol^2 and |dy| <= max_step, in fp64 of the float centroids without FMA,
 *     each operation rounded on its own (tol^2 = (double)tol * (double)tol).  A horizontal distance with a step bound:
 *     a ramp within the slope limit joins, a kerb up to max_step joins, a table top or a car roof does not.
 *   patch: a connected component of the candidates with size >= min_size.  Rank, ids, records (loam_b200_segment),
 *     the fp64 chunk sums and LOAM_B200_ERR_CAPACITY are dense_segment's, with the target index as the entry index
 *     (first, ties).  labels[i] (may be NULL): per target voxel in key order, its patch id or -1.
 *   product: the ground flags (a voxel is ground when it lies in a patch), stored with the target on LOAM_B200_OK and
 *     on LOAM_B200_ERR_CAPACITY (capacity only limits the records written).  A later dense_ground replaces them; a
 *     target build, load or release drops them, like the ray index, distance field and place database.
 *   Limitation: a large flat upward surface with no step to the street, such as a rooftop, is a patch like the street;
 *     its records' lo[1] / hi[1] let the caller reject it by height.
 *   LOAM_B200_ERR_ARG: tol or max_step not finite and > 0, max(tol, max_step) / leaf > 4 (r <= 5, as dense_segment),
 *   max_slope_deg outside [0, 90), max_curvature NaN or negative, min_size < 1, cap < 0, a NULL params or n_out,
 *   NULL patches with cap > 0.  LOAM_B200_ERR_STATE without a target.
 * dense_segment_above_ground: dense_segment's arguments, semantics, records, ranking and errors over the entries that
 *   are not ground (a voxel of a patch dropped by min_size is an entry); entry indices, first and ties are target
 *   indices; labels cover the whole target in key order, -1 for a ground voxel.  When no voxel is ground it equals
 *   dense_segment bit for bit.  LOAM_B200_ERR_STATE without a target or without ground flags.
 * dense_ground_cloud: per point p of xyzi (n float[4], w ignored; host memory, or device memory when on_device != 0):
 *   q = pointAssociateToMap(pose, p) as dense_align_iterate computes it (fp32, no FMA); its match is the alignment's
 *   rule restricted to the ground voxels (the first smallest d2 among the ground voxels of q's search_radius box,
 *   accepted when d2 < gate, gate = s * s, s = (float)search_radius * leaf); the point is ground when it has a match
 *   and |pd| <= max_height, pd = (nx*(qx - cx) + ny*(qy - cy)) + nz*(qz - cz) in fp32.
 *   labels (host, may be NULL): int8 per point, 1 ground, 0 not ground, -1 not finite or q's voxel outside the key
 *   range.  nonground (may be NULL; host memory when on_device == 0, device memory otherwise, so that it can go
 *   straight into cloud_segment with on_device = 1): the points labelled 0 in input order, room for n points needed.
 *   *n_nonground: their number.  LOAM_B200_ERR_ARG: dense_align_iterate's (n < 0, NULL xyzi with n > 0, a NULL or
 *   non-finite pose, search_radius outside 1..3), max_height not finite or negative, NULL n_nonground.
 *   LOAM_B200_ERR_STATE without a target or without ground flags.
 * Every argument check runs on the host before anything is launched, so a refused call changes nothing.  Launches,
 * with seg(m) = dense_segment's launches for a target of m voxels (0 for m = 0): dense_ground 5 + seg(candidates);
 * dense_segment_above_ground 4 + seg(entries); dense_ground_cloud 3, plus 1 with nonground; none for an empty target
 * or cloud.
 * ------------------------------------------------------------------------------------------------------------------ */
typedef struct {
  float max_slope_deg;  /* the steepest normal tilt from y that is still ground, [0, 90) */
  float max_curvature;  /* the largest curvature (normal w) that is still ground; +inf: no curvature test */
  float tol;            /* horizontal joining distance, metres */
  float max_step;       /* largest height step between joined voxels, metres */
  int min_size;         /* voxels of the smallest patch kept as ground */
} loam_b200_ground_params;

int loam_b200_dense_ground(loam_b200_ctx* ctx, const loam_b200_ground_params* params, int32_t* labels,
                           loam_b200_segment* patches, int cap, int* n_out);
int loam_b200_dense_segment_above_ground(loam_b200_ctx* ctx, float tol, int min_size, int max_size, int32_t* labels,
                                         loam_b200_segment* segments, int cap, int* n_out);
int loam_b200_dense_ground_cloud(loam_b200_ctx* ctx, const float* xyzi, int n, int on_device,
                                 const loam_b200_pose* pose, int search_radius, float max_height, int8_t* labels,
                                 float* nonground, int* n_nonground);

/* ------------------------------------------------------------------------------------------------------------------
 * Multi-GPU (one process per GPU).  With a shard set, loam_b200_map_iterate evaluates this rank's contiguous slice
 * of the corner and surface queries; with a communicator the 32-float partial normal equations are all-reduced
 * (NCCL, sum, fp32) on the context's stream directly behind the kernel, so every rank returns the same totals and
 * runs the same 6x6 solve.  rank 0 creates the id, the caller distributes it (torch.distributed, MPI, a file, ...).
 * ------------------------------------------------------------------------------------------------------------------ */
int loam_b200_comm_unique_id(unsigned char out[128]);
int loam_b200_comm_init(loam_b200_ctx* ctx, int rank, int world, const unsigned char id[128]);
int loam_b200_comm_destroy(loam_b200_ctx* ctx);
/* slice only, no collective: loam_b200_map_iterate returns PARTIAL sums for the caller to reduce */
int loam_b200_map_set_shard(loam_b200_ctx* ctx, int rank, int world);

/* ------------------------------------------------------------------------------------------------------------------
 * Kernel timing (CUDA events on the context's stream) for bench.py's roofline: accumulated GPU milliseconds and
 * launch counts per kernel family since the last reset.
 * ------------------------------------------------------------------------------------------------------------------ */
enum { LOAM_B200_K_FEATURES = 0, LOAM_B200_K_TREE_BUILD = 1, LOAM_B200_K_KNN = 2, LOAM_B200_K_MAP_ITER = 3,
       LOAM_B200_K_ODOM_ITER = 4, LOAM_B200_K_TRANSFORM = 5, LOAM_B200_K_VOXEL = 6, LOAM_B200_K_DENSE = 7,
       LOAM_B200_NUM_KERNEL_FAMILIES = 8 };
int loam_b200_profile_enable(loam_b200_ctx* ctx, int on);
int loam_b200_profile_reset(loam_b200_ctx* ctx);
int loam_b200_profile_get(loam_b200_ctx* ctx, int family, double* gpu_ms, long long* launches);
/* total kernel launches issued by this context since creation */
long long loam_b200_launch_count(loam_b200_ctx* ctx);
/* ... by every context of this process */
long long loam_b200_total_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif /* LOAM_B200_H */
