/* loam_b200_host.h -- C handles over the C++ drop-in classes loam::BasicScanRegistration / BasicLaserOdometry /
 * BasicLaserMapping (the headers under loam_velodyne_b200/csrc/host/loam_velodyne/), for callers that cannot include C++ headers
 * (the Python package, bench.py, ctypes tests).  C++ callers -- including the reference's ROS adapters, which derive
 * from the Basic* classes (ScanRegistration.h:55, LaserOdometry.h:56, LaserMapping.h:54 upstream) -- use the classes
 * directly.
 *
 * Points are packed float[4] = (x, y, z, intensity); twists are float[6] = (rot_x, rot_y, rot_z, pos.x, pos.y, pos.z).
 * Functions returning int give 0 on success and a negative value on failure; loam_b200_host_last_error() has the text
 * (per thread).  A failure here is always loud: there is no CPU fallback behind these handles.
 */
#ifndef LOAM_B200_HOST_H
#define LOAM_B200_HOST_H

#include "loam_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

const char* loam_b200_host_last_error(void);
/* CUDA device used by objects created afterwards (default: $LOAM_B200_DEVICE, else $LOCAL_RANK, else 0) */
void loam_b200_host_set_device(int device);

/* The 6 x 6 Gauss-Newton step of both loops (BasicLaserOdometry.cpp:559-600, BasicLaserMapping.cpp:867-908) as the
 * library solves it on host and device (csrc/lmstep.cuh: gn_solve): x = colPivHouseholderQr(AtA).solve(AtB); on the first
 * iteration eigenvalues of AtA below eigen_threshold switch the degeneracy projection on.  Pure host arithmetic (no GPU):
 * exposed for the parity tests.  AtA row-major 36 floats; *degenerate_out receives 0 / 1. */
int loam_b200_host_gn_solve(const float* AtA, const float* AtB, int first_iteration, float eigen_threshold, float* x_out6,
                            int* degenerate_out);

/* ---- loam::BasicTransformMaintenance (host-only pose fusion, BasicTransformMaintenance.cpp:45-178) ----
 * sum / bef / aft: rot_x, rot_y, rot_z, x, y, z of the odometry pose, the odometry pose at the last mapping update and the
 * mapped pose of that update (updateOdometry + updateMappingTransform); mapped_out6 = transformMapped() after
 * transformAssociateToMap(). */
int loam_b200_transform_maintenance(const float* sum6, const float* bef6, const float* aft6, float* mapped_out6);

/* ---- loam::BasicScanRegistration ---- */
void* loam_b200_scanreg_create(void);
void loam_b200_scanreg_destroy(void* h);
int loam_b200_scanreg_configure(void* h, float scanPeriod, int nFeatureRegions, int curvatureRegion, int maxCornerSharp,
                                int maxSurfaceFlat, float lessFlatFilterSize, float surfaceCurvatureThreshold);
/* processScanlines: ring r = ring_sizes[r] consecutive points */
int loam_b200_scanreg_process(void* h, const float* pts, const int* ring_sizes, int n_rings);
/* processUnorderedSweep: MultiScanRegistration::process (MultiScanRegistration.cpp:160-238) -- n unordered sensor-frame
 * xyz points (3 floats each) binned into rings on the GPU with MultiScanMapper(lower, upper, n_rings), then extraction */
int loam_b200_scanreg_process_unordered(void* h, const float* xyz, int n, float lower_bound_deg, float upper_bound_deg,
                                        int n_rings);
/* which: 0 laserCloud, 1 cornerPointsSharp, 2 cornerPointsLessSharp, 3 surfacePointsFlat, 4 surfacePointsLessFlat */
int loam_b200_scanreg_cloud_size(void* h, int which);
int loam_b200_scanreg_cloud_copy(void* h, int which, float* out);
/* which: 1 sharp, 2 less sharp, 3 flat -> indices into laserCloud */
int loam_b200_scanreg_index_size(void* h, int which);
int loam_b200_scanreg_index_copy(void* h, int which, int* out);

/* ---- loam::BasicLaserOdometry ---- */
void* loam_b200_odom_create(float scanPeriod, int maxIterations);
void loam_b200_odom_destroy(void* h);
int loam_b200_odom_set_inputs(void* h, const float* sharp, int n_sharp, const float* less_sharp, int n_less_sharp,
                              const float* flat, int n_flat, const float* less_flat, int n_less_flat,
                              const float* full, int n_full);
int loam_b200_odom_process(void* h);
int loam_b200_odom_full_to_end(void* h); /* transformToEnd(laserCloud()), as LaserOdometry::publishResult does */
/* which: 0 transform, 1 transformSum */
int loam_b200_odom_get_twist(void* h, int which, float* out6);
/* which: 0 lastCornerCloud, 1 lastSurfaceCloud, 2 laserCloud */
int loam_b200_odom_cloud_size(void* h, int which);
int loam_b200_odom_cloud_copy(void* h, int which, float* out);
int loam_b200_odom_last_iterations(void* h);

/* ---- loam::BasicLaserMapping ---- */
void* loam_b200_map_create(float scanPeriod, int maxIterations);
void loam_b200_map_destroy(void* h);
int loam_b200_map_seed(void* h, const float* corner, int n_corner, const float* surf, int n_surf);
int loam_b200_map_set_inputs(void* h, const float* corner_last, int n_corner, const float* surf_last, int n_surf,
                             const float* full, int n_full);
int loam_b200_map_update_odometry(void* h, const float* sum6);
int loam_b200_map_process(void* h); /* 1 processed, 0 frame skipped, <0 error */
/* which: 0 transformAftMapped, 1 transformBefMapped, 2 transformTobeMapped */
int loam_b200_map_get_twist(void* h, int which, float* out6);
/* which: 0 laserCloud (registered), 1 laserCloudSurroundDS, 2 cornerFromMap, 3 surfFromMap, 4 cornerStackDS,
 *        5 surfStackDS, 6 all corner cubes, 7 all surf cubes */
int loam_b200_map_cloud_size(void* h, int which);
int loam_b200_map_cloud_copy(void* h, int which, float* out);
int loam_b200_map_last_iterations(void* h);
/* host wall seconds of the last process(): begin_sweep, LM loop, end_sweep, surround map */
int loam_b200_map_last_phase_seconds(void* h, double* out4);
/* measurement hook: the scan-to-map iteration kernel exactly as this object launches it (own context, persistent map, the
 * queries of the last process()), CUDA-event time over `reps` launches at the current pose.  out5 = average launch
 * microseconds, queries, table probes / query, candidate points / query, selected correspondences */
int loam_b200_map_kernel_profile(void* h, int reps, double* out5);
/* ... on n caller-supplied surface queries (packed float4, map frame, identity pose) against this object's persistent map:
 * the k-NN bandwidth stress (queries spread over a map far larger than L2).  Replaces the queries of the last process(). */
int loam_b200_map_kernel_profile_queries(void* h, const float* queries, int n, int reps, double* out5);
/* test hook: keep a copy of laserCloudCornerFromMap / laserCloudSurfFromMap (cloud ids 2, 3) at every process() */
int loam_b200_map_retain_from_map(void* h, int on);
/* whole-run voxel map (BasicLaserMapping::enableDenseMap & co., include/loam_b200.h "Whole-run voxel map"):
 * stats out3 = voxels, skipped points, dropped points; export writes n_out packed float[4] centroids (+ counts when
 * counts != NULL) in ascending voxel order, LOAM_B200_ERR_CAPACITY (with *n_out set) when they exceed cap.  On a
 * streaming pipeline's mapping object these four return LOAM_B200_ERR_STATE while sweeps are in flight, i.e. from
 * loam_b200_pipeline_submit until loam_b200_pipeline_collect has returned that sweep's result. */
int loam_b200_map_dense_enable(void* h, float leaf, long long max_voxels);
int loam_b200_map_dense_stats(void* h, long long* out3);
int loam_b200_map_dense_export(void* h, float* xyzi, unsigned int* counts, int cap, int* n_out);
int loam_b200_map_dense_clear(void* h);
/* visibility pass (BasicLaserMapping::enableDenseVisibility, include/loam_b200.h "loam_b200_dense_visibility") and the
 * export filtered by max_miss_ratio (BasicLaserMapping::denseMapFiltered): as loam_b200_map_dense_export,
 * plus per-voxel hits / misses when non-NULL.  Same in-flight rule as the four above. */
int loam_b200_map_dense_visibility(void* h, double h_res_deg, double v_res_deg, double margin);
/* carve mode of the pass (BasicLaserMapping::enableDenseCarving, include/loam_b200.h "loam_b200_dense_carving");
 * max_range 0 turns it off.  Same in-flight rule. */
int loam_b200_map_dense_carving(void* h, double margin, double max_range);
int loam_b200_map_dense_export_filtered(void* h, double max_miss_ratio, float* xyzi, unsigned int* counts,
                                        unsigned short* hits, unsigned short* misses, int cap, int* n_out);
/* the filtered export with a normal and curvature per voxel (BasicLaserMapping::denseMapNormals, include/loam_b200.h
 * "loam_b200_dense_export_normals"): normals float[4] (nx, ny, nz, curvature) per voxel in the centroids' order; same
 * arguments, capacity rule and in-flight rule as loam_b200_map_dense_export_filtered, viewpoint = 3 doubles. */
int loam_b200_map_dense_export_normals(void* h, double max_miss_ratio, int radius, const double* viewpoint,
                                       float* xyzi, unsigned int* counts, float* normals, int cap, int* n_out);
/* snapshots and merging (BasicLaserMapping::denseMapSnapshot / mergeDenseMap, include/loam_b200.h "Whole-run voxel
 * map snapshots and merging"), same in-flight rule.  snapshot: as loam_b200_dense_snapshot (keys, hits, misses may be
 * NULL; capacity rule of the exports).  merge: n entries as loam_b200_dense_merge, pose6 = twist (rot_x, rot_y, rot_z,
 * x, y, z) or NULL. */
int loam_b200_map_dense_snapshot(void* h, unsigned long long* keys, unsigned int* counts, unsigned short* hits,
                                 unsigned short* misses, double* sums, int cap, int* n_out);
int loam_b200_map_dense_merge(void* h, const unsigned int* counts, const unsigned short* hits,
                              const unsigned short* misses, const double* sums, int n, const float* pose6);
/* test query: loam_b200_debug_dense_table_slots of the mapping object's context (BasicLaserMapping::denseTableSlots) */
int loam_b200_map_debug_dense_table_slots(void* h, long long* out);
/* alignment against the whole-run map (BasicLaserMapping::buildDenseTarget / loadDenseTarget / alignToDenseTarget,
 * include/loam_b200.h "Alignment against the whole-run voxel map"), same in-flight rule as the exports above.
 * target_build: *n_out = the target's voxels, viewpoint = 3 doubles.  target_load: n entries of xyzi float[4] and
 * normals float[4] (nx, ny, nz, curvature).  align: n sensor-frame points, initial6 = twist; twist_out6 = the aligned
 * twist, stats_out4 = iterations, n_selected, degenerate, converged; *rms_out = the point-to-plane RMS (each out may be
 * NULL except twist_out6). */
int loam_b200_map_dense_target_build(void* h, double max_miss_ratio, int radius, const double* viewpoint, int* n_out);
int loam_b200_map_dense_target_load(void* h, float leaf, const float* xyzi, const float* normals, int n);
int loam_b200_map_dense_align(void* h, const float* xyzi, int n, const float* initial6, int search_radius,
                              int max_iterations, float* twist_out6, int* stats_out4, float* rms_out);
/* relocalisation against that target (BasicLaserMapping::scoreDenseTarget / alignToDenseTarget over a vector /
 * relocalizeInDenseTarget, include/loam_b200.h "Relocalisation against the whole-run voxel map"), same in-flight rule.
 * k twists of 6 floats each.  score: n_selected[k], sum_pd2_sq[k].  align_batch: per run h, twist_out6[6h..],
 * stats_out4[4h..] and rms_out[h] as align (stats_out4 and rms_out may be NULL).  relocalize: at most cap candidates
 * into out, *n_out = candidates written. */
int loam_b200_map_dense_score(void* h, const float* xyzi, int n, const float* poses6, int k, int search_radius,
                              int* n_selected, float* sum_pd2_sq);
int loam_b200_map_dense_align_batch(void* h, const float* xyzi, int n, const float* initial6, int k, int search_radius,
                                    int max_iterations, float* twist_out6, int* stats_out4, float* rms_out);
int loam_b200_map_dense_relocalize(void* h, const float* xyzi, int n, const float* hyps6, int k,
                                   const loam_b200_reloc_params* prm, loam_b200_reloc_candidate* out, int cap,
                                   int* n_out);
/* ray casting that target (BasicLaserMapping::raycastDenseTarget, include/loam_b200.h "Ray casting the whole-run voxel
 * map"), same in-flight rule: n sensor-frame rays of float[4] from the twist pose6 -> range[n], index[n] (may be
 * NULL). */
int loam_b200_map_dense_raycast(void* h, const float* rays, int n, const float* pose6, float min_range,
                                float max_range, float* range, int* index);
/* distance field of that target (BasicLaserMapping::buildDenseDistanceField / queryDenseDistance, include/loam_b200.h
 * "Distance field of the whole-run voxel map"), same in-flight rule: build over the box lo[3], dims[3] -> dist and sq
 * (nx * ny * nz each, either may be NULL); query n map-frame points of float[4] -> dist[n], grad[3n] (may be NULL). */
int loam_b200_map_dense_distance_build(void* h, const int* lo, const int* dims, float max_distance, float* dist,
                                       int* sq);
int loam_b200_map_dense_distance_query(void* h, const float* xyzi, int n, float* dist, float* grad);
/* place recognition and global relocalisation in that target (BasicLaserMapping::buildDensePlaces /
 * queryDensePlaces / relocalizeGlobalInDenseTarget, include/loam_b200.h "Place recognition and global
 * relocalisation"), same in-flight rule: k positions of float[3], n_rays rays and n points of float[4]. */
int loam_b200_map_dense_place_build(void* h, const float* positions, int k, const float* rays, int n_rays,
                                    const loam_b200_place_params* prm);
int loam_b200_map_dense_place_query(void* h, const float* xyzi, int n, int top_m, loam_b200_place_match* out,
                                    int* n_out);
int loam_b200_map_dense_relocalize_global(void* h, const float* xyzi, int n, int top_m, float yaw_step_deg,
                                          int yaw_steps, float xz_step, int xz_steps,
                                          const loam_b200_reloc_params* prm, loam_b200_reloc_candidate* out, int cap,
                                          int* n_out);
/* Euclidean segmentation of that target (BasicLaserMapping::segmentDenseTarget, include/loam_b200.h "Euclidean
 * segmentation of the whole-run voxel map and of clouds"), same in-flight rule: labels (may be NULL) receive one int
 * per target voxel, as many as loam_b200_map_dense_target_size (BasicLaserMapping::denseTargetSize) reports;
 * segments[0 .. *n_out), LOAM_B200_ERR_CAPACITY when *n_out > cap. */
int loam_b200_map_dense_target_size(void* h, int* n_out);
int loam_b200_map_dense_segment(void* h, float tol, int min_size, int max_size, int* labels,
                                loam_b200_segment* segments, int cap, int* n_out);
/* Ground of that target (BasicLaserMapping::groundDenseTarget / segmentDenseTargetAboveGround / splitGround,
 * include/loam_b200.h "Ground of the whole-run voxel map"), same in-flight rule and label / record conventions as
 * loam_b200_map_dense_segment.  ground_cloud: the points of xyzi (sensor frame, at pose6) labelled ground go to
 * ground[0 .. *n_ground), those labelled not ground to nonground[0 .. *n_nonground), each in input order (either
 * array may be NULL; room for n points each). */
int loam_b200_map_dense_ground(void* h, const loam_b200_ground_params* params, int* labels,
                               loam_b200_segment* patches, int cap, int* n_out);
int loam_b200_map_dense_segment_above_ground(void* h, float tol, int min_size, int max_size, int* labels,
                                             loam_b200_segment* segments, int cap, int* n_out);
int loam_b200_map_dense_ground_cloud(void* h, const float* xyzi, int n, const float* pose6, int search_radius,
                                     float max_height, float* ground, int* n_ground, float* nonground,
                                     int* n_nonground);
/* multi-GPU, one process per GPU: rank 0 calls loam_b200_host_nccl_unique_id and distributes the 128 bytes; every rank
 * then enables sharding on its mapping object (nccl_id128 = NULL: slice the queries only, no collective) */
int loam_b200_host_nccl_unique_id(unsigned char* out128);
int loam_b200_map_enable_sharding(void* h, int rank, int world, const unsigned char* nccl_id128);

/* multi-GPU with the MAP sharded by cube slabs along x (include/loam_b200.h "peer"): every rank exports its 64-byte inbox
 * handle, the caller all-gathers them, every rank enables sharding with all handles in rank order.  A rank then stores
 * only its slabs (+ 2 m halo; loam_b200_map_seed keeps the points that belong to it) and the per-iteration normal equations
 * are all-reduced inside the iteration kernel over NVLink peer memory.  _local: objects of one process, hs[r] = rank r. */
int loam_b200_map_peer_export(void* h, unsigned char* out64);
int loam_b200_map_enable_cube_sharding(void* h, int rank, int world, const unsigned char* handles, int slab_metres);
int loam_b200_map_enable_cube_sharding_local(void** hs, int world, int slab_metres);
/* unmap the peers' inboxes: every rank calls this and the ranks synchronise BEFORE any of them destroys its object (memory
 * exported over CUDA IPC must not be freed while another process still has it mapped) */
int loam_b200_map_disable_cube_sharding(void* h);

/* ---- the three chained in-process: registration -> odometry -> mapping on one sweep ---- */
void* loam_b200_pipeline_create(float scanPeriod, int odomMaxIter, int mapMaxIter);
void loam_b200_pipeline_destroy(void* h);
int loam_b200_pipeline_seed_map(void* h, const float* corner, int n_corner, const float* surf, int n_surf);
/* stage_seconds[5]: registration, odometry, full->end, mapping, total (steady_clock, host wall time) */
int loam_b200_pipeline_sweep(void* h, const float* pts, const int* ring_sizes, int n_rings, float* odom_sum6,
                             float* map_aft6, double* stage_seconds);
/* same, the sweep already resident in GPU memory (d_pts: device pointer to the packed points) */
int loam_b200_pipeline_sweep_device(void* h, const void* d_pts, const int* ring_sizes, int n_rings, float* odom_sum6,
                                    float* map_aft6, double* stage_seconds);
/* same chain, but every hand-off goes through host pcl clouds and the reference's own entry points
 * (processScanlines(vector<PointCloud>) / cloud Ptr accessors), as separate ROS nodes would use the classes */
int loam_b200_pipeline_sweep_hostclouds(void* h, const float* pts, const int* ring_sizes, int n_rings, float* odom_sum6,
                                        float* map_aft6, double* stage_seconds);
/* Streaming form: registration, odometry and mapping run as three concurrent single-threaded stages over consecutive
 * sweeps -- the way the reference's three ROS nodes run (CMakeLists.txt:40-50) -- connected by the device-to-device
 * hand-offs; results equal the sequential chain bit for bit.  submit() queues one sweep (host `pts` or device `d_pts`,
 * the other NULL; the buffer must stay valid until its result has been collected) and blocks only while two sweeps are
 * already waiting; collect() returns the oldest finished sweep: 1 = result written, 0 = nothing pending (or, with
 * wait == 0, nothing ready yet), -1 = a stage failed (loam_b200_host_last_error).  Do not mix with the _sweep calls
 * while sweeps are in flight. */
int loam_b200_pipeline_submit(void* h, const float* pts, const void* d_pts, const int* ring_sizes, int n_rings);
int loam_b200_pipeline_collect(void* h, int wait, float* odom_sum6, float* map_aft6, int* ok);
/* out9 = seconds the registration / odometry / mapping stage threads spent [0..2] working, [3..5] waiting for a neighbour
 * stage, [6..8] in the adopt() hand-offs since streaming started (or the last reset); call while no sweep is in flight */
int loam_b200_pipeline_stage_seconds(void* h, double* out9, int reset);
/* wait until everything the three stage objects enqueued (or posted to their helper threads) has finished on the GPU */
int loam_b200_pipeline_sync(void* h);
void* loam_b200_pipeline_scanreg(void* h);
void* loam_b200_pipeline_odom(void* h);
void* loam_b200_pipeline_map(void* h);

#ifdef __cplusplus
}
#endif
#endif
