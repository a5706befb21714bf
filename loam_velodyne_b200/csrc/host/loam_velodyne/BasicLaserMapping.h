// loam::BasicLaserMapping -- drop-in for upstream include/loam_velodyne/BasicLaserMapping.h:77-111.
// Same constructor, process(Time), updateIMU, updateOdometry (both overloads), mutable cloud references
// (laserCloud / laserCloudCornerLast / laserCloudSurfLast), downSizeFilter*() handles, setters / getters,
// transformAftMapped / transformBefMapped / laserCloudSurroundDS / hasFreshMap.
// The scan-to-map optimisation (optimizeTransformTobeMapped, BasicLaserMapping.cpp:626-926 upstream) runs its
// per-point work on the GPU: BVH build over the surrounding-map clouds, fused 5-NN + fit + Jacobian + normal-equation
// reduction per iteration; the host keeps the 6x6 solve and the O(1) pose algebra.
#pragma once

#include <cstdint>
#include <vector>

#include <pcl/filters/voxel_grid.h>
#include <pcl/point_cloud.h>
#include <pcl/point_types.h>

#include "Twist.h"
#include "time_utils.h"

namespace loam {

namespace b200 { class Context; class DualCloud; struct GaussNewtonSolver; }
class BasicLaserOdometry;

typedef struct IMUState2 {
  Time stamp;
  Angle roll;
  Angle pitch;
  static void interpolate(const IMUState2& start, const IMUState2& end, const float& ratio, IMUState2& result) {
    const float invRatio = 1 - ratio;
    result.roll = start.roll.rad() * invRatio + end.roll.rad() * ratio;
    result.pitch = start.pitch.rad() * invRatio + end.pitch.rad() * ratio;
  }
} IMUState2;

class BasicLaserMapping {
 public:
  explicit BasicLaserMapping(const float& scanPeriod = 0.1, const size_t& maxIterations = 10);
  ~BasicLaserMapping();
  BasicLaserMapping(const BasicLaserMapping&) = delete;
  BasicLaserMapping& operator=(const BasicLaserMapping&) = delete;

  bool process(Time const& laserOdometryTime);
  void updateIMU(IMUState2 const& newState);
  void updateOdometry(double pitch, double yaw, double roll, double x, double y, double z);
  void updateOdometry(Twist const& twist);

  // input clouds (filled by the caller, LaserMapping.cpp:177-200 upstream) / registered full-resolution output;
  // the authoritative copies live in HBM, these handles download on first use and mark the GPU copy stale
  pcl::PointCloud<pcl::PointXYZI>& laserCloud();
  pcl::PointCloud<pcl::PointXYZI>& laserCloudCornerLast();
  pcl::PointCloud<pcl::PointXYZI>& laserCloudSurfLast();

  void setScanPeriod(float val) { _scanPeriod = val; }
  void setMaxIterations(size_t val) { _maxIterations = val; }
  void setDeltaTAbort(float val) { _deltaTAbort = val; }
  void setDeltaRAbort(float val) { _deltaRAbort = val; }

  auto& downSizeFilterCorner() { return _downSizeFilterCorner; }
  auto& downSizeFilterSurf() { return _downSizeFilterSurf; }
  auto& downSizeFilterMap() { return _downSizeFilterMap; }

  auto frameCount() const { return _frameCount; }
  auto scanPeriod() const { return _scanPeriod; }
  auto maxIterations() const { return _maxIterations; }
  auto deltaTAbort() const { return _deltaTAbort; }
  auto deltaRAbort() const { return _deltaRAbort; }

  auto const& transformAftMapped() const { return _transformAftMapped; }
  auto const& transformBefMapped() const { return _transformBefMapped; }
  pcl::PointCloud<pcl::PointXYZI> const& laserCloudSurroundDS() const;

  bool hasFreshMap() const { return _downsizedMapCreated; }

  // extensions (not in the reference API): pre-seed the cube map with points given in the map frame, using the same
  // cube-index arithmetic as the insertion step (upstream BasicLaserMapping.cpp:540-553); introspection for tests.
  void seedMap(pcl::PointCloud<pcl::PointXYZI> const& cornerPoints, pcl::PointCloud<pcl::PointXYZI> const& surfPoints);
  size_t lastIterationCount() const { return _lastIterations; }
  // sizes of the down-sized feature stacks of the last process() (the queries of its optimisation loop)
  size_t cornerStackSize() const { return (size_t)_mapSizes[2]; }
  size_t surfStackSize() const { return (size_t)_mapSizes[3]; }
  // host wall seconds of the last process(): begin_sweep, LM loop, end_sweep, surround map
  const double* lastPhaseSeconds() const { return _phase; }
  auto const& transformTobeMapped() const { return _transformTobeMapped; }
  pcl::PointCloud<pcl::PointXYZI> const& cornerStackDS() const;
  pcl::PointCloud<pcl::PointXYZI> const& surfStackDS() const;
  pcl::PointCloud<pcl::PointXYZI> const& cornerFromMap() const;
  pcl::PointCloud<pcl::PointXYZI> const& surfFromMap() const;
  void collectMap(pcl::PointCloud<pcl::PointXYZI>& corner, pcl::PointCloud<pcl::PointXYZI>& surf) const;
  // take last corner / last surface / full-resolution clouds and transformSum from an odometry object without a
  // host round trip (LaserOdometry::publishResult -> LaserMapping::*Handler upstream)
  void adopt(BasicLaserOdometry& odom);
  b200::Context* deviceContext() { return _gpu; }
  // multi-GPU (one process per GPU): this object evaluates the rank-th of `world` slices of the correspondences and
  // all-reduces the 6x6 normal equations over NCCL every iteration (ncclId: 128 bytes from
  // loam_b200_comm_unique_id on rank 0; nullptr = slice only, the caller reduces)
  void enableSharding(int rank, int world, const unsigned char* ncclId);
  // multi-GPU with the MAP sharded by cube slabs (one process per GPU; csrc/shard.cuh, include/loam_b200.h "peer"):
  // exportPeerHandle() gives this rank's 64-byte inbox handle, enableCubeSharding() takes all of them in rank order.
  // Afterwards this object stores only the slabs it owns (+ 2 m halo): seedMap() keeps the points that belong here,
  // process() evaluates the queries that fall into its slabs and the per-iteration normal equations are all-reduced
  // inside the iteration kernel over NVLink peer memory.  slabMetres: slab width (whole metres, default 10).
  void exportPeerHandle(unsigned char out64[64]);
  void enableCubeSharding(int rank, int world, const unsigned char* handles, int slabMetres = 10);
  // the same for several objects of ONE process (tests / single-process multi-GPU): objs[r] becomes rank r
  static void enableCubeShardingLocal(BasicLaserMapping** objs, int world, int slabMetres = 10);
  /** Test hook (not in the reference): keep a copy of the points of the cubes in view (upstream's internal
   *  _laserCloudCornerFromMap / _laserCloudSurfFromMap) after every process(); off by default, the persistent GPU map
   *  only needs their sizes. */
  void retainFromMapClouds(bool on);

  // extension (not in the reference API): the whole-run voxel map.  Once enabled, every process() that returns true adds
  // the registered full-resolution cloud (laserCloud() in the map frame) to a voxel map on the GPU that is never rolled
  // or pruned, unlike the 21 x 11 x 21 cube grid.  Per voxel: point count and the centroid of x, y, z and intensity
  // (fp64 sums), exported in ascending voxel order (pcl::VoxelGrid's order: x fastest, then y, then z).  At most
  // maxVoxels voxels are kept: once full, new voxels are refused (their points counted as dropped) while the kept ones
  // keep accumulating.  Off by default; throws on a sharded object and on another leaf while the map holds voxels.
  struct DenseMapStats { long long voxels, skipped, dropped; };
  void enableDenseMap(float leaf, long long maxVoxels = 2147483647ll);
  DenseMapStats denseMapStats();
  void denseMap(pcl::PointCloud<pcl::PointXYZI>& out, std::vector<uint32_t>* counts = nullptr);
  void clearDenseMap();
  // Visibility pass over the whole-run map (off by default; include/loam_b200.h "loam_b200_dense_visibility"): every
  // process() first renders its registered cloud as a range image (hRes x vRes degree pixels, minimum range) from the
  // optimised pose and counts a miss for every stored voxel that lies more than `margin` metres in front of the return
  // in its pixel.  hRes = 0 turns it off; throws without the dense map and on bad arguments.
  void enableDenseVisibility(double hRes, double vRes, double margin);
  // Carve mode of that pass (off by default; include/loam_b200.h "loam_b200_dense_carving"): every process() walks each
  // registered point's ray from the optimised pose through the map and counts one miss for every stored voxel a ray
  // crosses more than `margin` metres short of its return (up to maxRange) that no point of the sweep falls into.
  // maxRange = 0 turns it off; throws without the dense map, on bad arguments and while the range-image mode is on.
  void enableDenseCarving(double margin, double maxRange);
  // the voxels with misses <= maxMissRatio * hits (a voxel's hits: the sweeps that put points into it); +inf returns
  // every voxel, as denseMap above.  hits / misses: per-voxel evidence counters (saturating at 65535) when non-null.
  void denseMapFiltered(pcl::PointCloud<pcl::PointXYZI>& out, double maxMissRatio,
                        std::vector<uint32_t>* counts = nullptr, std::vector<uint16_t>* hits = nullptr,
                        std::vector<uint16_t>* misses = nullptr);
  // the voxels of denseMapFiltered(maxMissRatio) with a surface normal and curvature each (include/loam_b200.h
  // "loam_b200_dense_export_normals"): pcl::NormalEstimation over the exported centroids with a box neighbourhood of
  // `radius` (1..3) voxels on every axis, normals flipped towards `viewpoint` (map frame; PCL's default, the origin, is
  // the first sweep's sensor position).  Fewer than 3 neighbours: NaN normal and curvature.  Throws on bad arguments.
  void denseMapNormals(pcl::PointCloud<pcl::PointXYZINormal>& out, double maxMissRatio, int radius,
                       const Vector3& viewpoint, std::vector<uint32_t>* counts = nullptr);
  // the same with the viewpoint in double (x, y, z)
  void denseMapNormals(pcl::PointCloud<pcl::PointXYZINormal>& out, double maxMissRatio, int radius,
                       const double viewpoint[3], std::vector<uint32_t>* counts = nullptr);
  /** Test hook (not in the reference): slots of the whole-run map's hash table (0 while the map is off). */
  long long denseTableSlots();
  // Snapshots and merging of the whole-run map (include/loam_b200.h "Whole-run voxel map snapshots and merging"):
  // denseMapSnapshot gives every stored voxel's exact state in ascending key order (sums: x, y, z, intensity per voxel,
  // fp64); mergeDenseMap adds a snapshot into this map, as stored (pose nullptr) or under a rigid transform (e.g. the
  // pose of another session's first sweep found by relocalizeInDenseTarget).  Each entry's voxel follows from its
  // centroid at this map's leaf, so a snapshot of a finer map merges into a coarser one.  Resume a stopped run by
  // merging its snapshot into an empty map of the same leaf: the result is the snapshot bit for bit.  Throws on a
  // refused call (an entry with count 0 or hits 0, a sum or pose that is not finite, no dense map).
  struct DenseMapSnapshot {
    float leaf = 0.f;
    std::vector<uint64_t> keys;
    std::vector<uint32_t> counts;
    std::vector<uint16_t> hits, misses;
    std::vector<double> sums;  // 4 per voxel
  };
  void denseMapSnapshot(DenseMapSnapshot& out);
  void mergeDenseMap(const DenseMapSnapshot& snap, const Twist* pose = nullptr);
  // Alignment against the whole-run map (include/loam_b200.h "Alignment against the whole-run voxel map"): point-to-plane
  // Gauss-Newton of a sensor-frame cloud against a target of voxel centroids and normals on the GPU -- relocalisation
  // in a map built earlier, drift checks of a mapped pose, another sensor's or session's sweeps in the same map.
  // buildDenseTarget snapshots denseMapNormals(maxMissRatio, radius, viewpoint) as the target and returns its voxel
  // count; loadDenseTarget takes one from a saved cloud (a NaN normal_x: no normal; throws on entries outside the key
  // range or two in one voxel).  alignToDenseTarget runs the mapping stage's loop (skip below 50 correspondences,
  // eigenvalue threshold 100, deltaR 0.05 deg / deltaT 0.05 cm) from `initial`; refine coarse to fine by calling it
  // with searchRadius 3, then 1 from the first result.  The result never changes this object's poses or maps.
  struct DenseAlignResult {
    Twist pose;
    size_t iterations;  // executed (0: empty cloud or empty target)
    size_t nSelected;   // correspondences of the last executed iteration, at its input pose
    float rms;          // their point-to-plane RMS (metres)
    bool degenerate;    // the degeneracy projection was in effect
    bool converged;     // stopped by the thresholds, not by maxIterations
  };
  size_t buildDenseTarget(double maxMissRatio, int radius, const Vector3& viewpoint);
  size_t buildDenseTarget(double maxMissRatio, int radius, const double viewpoint[3]);
  void loadDenseTarget(float leaf, const pcl::PointCloud<pcl::PointXYZINormal>& target);
  DenseAlignResult alignToDenseTarget(const pcl::PointCloud<pcl::PointXYZI>& cloud, const Twist& initial,
                                      int searchRadius, int maxIterations);
  // Relocalisation against the target (include/loam_b200.h "Relocalisation against the whole-run voxel map"), for a
  // restart or a tracking loss with a rough position and no heading.  scoreDenseTarget: per pose the correspondences
  // and the sum of squared point-to-plane residuals of one alignment iteration there, all poses in one GPU pass.  The
  // vector overload of alignToDenseTarget runs one independent alignment per initial pose, each equal to the single
  // call.  relocalizationGrid: a yaw x (x, z) grid around a prior (y is up).  relocalizeInDenseTarget scores the
  // hypotheses, refines the `keep` best coarse to fine, scores them again, ranks and drops duplicates; candidate 0 is
  // the answer and its gap to candidate 1 the ambiguity.  Defaults of RelocParams are the recommended parameters.
  struct DenseScore {
    size_t nSelected;
    float sumPd2Sq;
  };
  struct RelocParams {
    RelocParams()
        : scoreRadius(3), coarseRadius(3), fineRadius(1), keep(16), maxIterations(30), dedupMetres(0.5f),
          dedupDegrees(5.0f) {}
    int scoreRadius, coarseRadius, fineRadius;
    int keep;
    int maxIterations;
    float dedupMetres, dedupDegrees;
  };
  struct RelocCandidate {
    size_t hypothesis;     // index into the hypotheses given
    size_t scoreSelected;  // correspondences at the hypothesis in the first score
    DenseAlignResult coarse, fine;  // fine.pose is the candidate's pose
    size_t selected;       // correspondences at fine.pose (fine radius)
    float rms;             // their point-to-plane RMS
    const Twist& pose() const { return fine.pose; }
  };
  std::vector<DenseScore> scoreDenseTarget(const pcl::PointCloud<pcl::PointXYZI>& cloud,
                                           const std::vector<Twist>& poses, int searchRadius);
  std::vector<DenseAlignResult> alignToDenseTarget(const pcl::PointCloud<pcl::PointXYZI>& cloud,
                                                   const std::vector<Twist>& initial, int searchRadius,
                                                   int maxIterations);
  std::vector<RelocCandidate> relocalizeInDenseTarget(const pcl::PointCloud<pcl::PointXYZI>& cloud,
                                                      const std::vector<Twist>& hypotheses,
                                                      const RelocParams& params = RelocParams(),
                                                      size_t maxCandidates = 16);
  // defaults (the recommended grid): full circle at 2 deg, 0.4 m steps four to each side of the prior (14661 poses)
  static std::vector<Twist> relocalizationGrid(const Twist& prior, float yawStepDeg = 2.0f, int yawSteps = 90,
                                               float xzStep = 0.4f, int xzSteps = 4);
  // Ray casting the target (include/loam_b200.h "Ray casting the whole-run voxel map"): what the sensor should see
  // from `pose`.  Each point of `rays` is a direction in the sensor frame (a sweep's own points may be passed); range[i]
  // is the surfel-refined distance to the first target voxel the ray meets within (minRange, maxRange], +inf when
  // none; index (optional) its position in the target, -1 when none.
  void raycastDenseTarget(const pcl::PointCloud<pcl::PointXYZI>& rays, const Twist& pose, float minRange,
                          float maxRange, std::vector<float>& range, std::vector<int>* index = nullptr);
  // Distance field of the target (include/loam_b200.h "Distance field of the whole-run voxel map"): exact distances to
  // the nearest target voxel in the box of voxels lo + [0, dims), kept on the device.  dist / sq (optional) receive
  // the box's float distances (+inf beyond maxDistance) and squared voxel distances (-1 beyond), x fastest.
  // queryDenseDistance interpolates the field at map-frame points: dist per point (NaN outside the box's cell
  // centres) and, optionally, its gradient (3 floats per point).
  void buildDenseDistanceField(const int lo[3], const int dims[3], float maxDistance, std::vector<float>* dist = nullptr,
                               std::vector<int>* sq = nullptr);
  void queryDenseDistance(const pcl::PointCloud<pcl::PointXYZI>& points, std::vector<float>& dist,
                          std::vector<float>* grad = nullptr);
  // Place recognition and global relocalisation (include/loam_b200.h "Place recognition and global relocalisation"),
  // for a cloud with no prior pose.  buildDensePlaces renders a polar height descriptor at each position from the
  // target through the ray cast (rays: a sensor's directions); the database lives with the target.  queryDensePlaces
  // compares the cloud's descriptor with every place over every heading -> the topM best, each with its heading.
  // relocalizeGlobalInDenseTarget refines those places with relocalizeInDenseTarget over a small grid around each;
  // a candidate's hypothesis / grid size is its place's rank.  Defaults are the recommended parameters.
  struct PlaceParams {
    PlaceParams() : rings(20), sectors(60), maxRadius(80.f), heightOffset(2.f), minRange(0.f), maxRange(100.f) {}
    int rings, sectors;
    float maxRadius, heightOffset;
    float minRange, maxRange;  // the database's ray cast
  };
  struct PlaceMatch {
    size_t candidate;  // index into the positions of buildDensePlaces
    int shift;         // the best sector shift
    float yaw;         // its heading (rot_y), in (-pi, pi]
    Vector3 position;  // the place's position
    double dist;       // descriptor distance (0: identical up to the shift)
  };
  struct GlobalGrid {
    GlobalGrid() : topM(5), yawStepDeg(2.f), yawSteps(3), xzStep(0.4f), xzSteps(5) {}
    int topM;
    float yawStepDeg;
    int yawSteps;
    float xzStep;
    int xzSteps;
  };
  void buildDensePlaces(const std::vector<Vector3>& positions, const pcl::PointCloud<pcl::PointXYZI>& rays,
                        const PlaceParams& params = PlaceParams());
  std::vector<PlaceMatch> queryDensePlaces(const pcl::PointCloud<pcl::PointXYZI>& cloud, size_t topM = 5);
  std::vector<RelocCandidate> relocalizeGlobalInDenseTarget(const pcl::PointCloud<pcl::PointXYZI>& cloud,
                                                            const GlobalGrid& grid = GlobalGrid(),
                                                            const RelocParams& params = RelocParams(),
                                                            size_t maxCandidates = 16);
  // Euclidean segmentation of the target (include/loam_b200.h "Euclidean segmentation of the whole-run voxel map and
  // of clouds"; pcl::EuclideanClusterExtraction over the target's voxels, exact): connected components of the voxels
  // whose centroids lie within `tolerance` metres (at most 4 leaves), kept when their size is in [minSize, maxSize],
  // ranked by size descending (ties: smallest voxel index first).  labels (optional): per target voxel, in the
  // target's order (raycastDenseTarget's index), its segment's rank or -1.  Throws without a target and on bad
  // arguments.
  struct DenseSegment {
    size_t size;         // voxels
    size_t first;        // the smallest target index among them
    float lo[3], hi[3];  // min / max of their centroids per axis
    float centroid[3];   // mean of their centroids
  };
  // voxels of the current target (the length of segmentDenseTarget's labels); throws without a target
  size_t denseTargetSize();
  std::vector<DenseSegment> segmentDenseTarget(float tolerance, int minSize = 1, int maxSize = 2147483647,
                                               std::vector<int>* labels = nullptr);
  // Ground of the target (include/loam_b200.h "Ground of the whole-run voxel map"; y is up).  groundDenseTarget:
  // patches of voxels whose normal lies within maxSlopeDeg of y and whose curvature is at most maxCurvature (+inf: no
  // curvature test), joined within `tolerance` metres horizontally and `maxStep` metres vertically, kept from minSize
  // voxels; ranked and recorded as segmentDenseTarget.  The ground flags stay with the target (until its next build
  // or load) for the two calls below.  A flat roof with no step to the street is a patch too: reject it by lo[1].
  // segmentDenseTargetAboveGround: segmentDenseTarget over the voxels that are not ground (labels -1 on the ground).
  // splitGround: the points of a sensor-frame cloud at `pose` that lie within maxHeight of a ground voxel's plane
  // (its nearest ground centroid within searchRadius voxels) go to `ground`, the other finite points to `nonGround`,
  // both in input order.  All throw without a target or ground and on bad arguments.
  struct DenseGroundParams {
    DenseGroundParams() : maxSlopeDeg(15.f), maxCurvature(0.05f), tolerance(0.3f), maxStep(0.2f), minSize(200) {}
    float maxSlopeDeg, maxCurvature;  // degrees from y; the normal's w (+inf: no curvature test)
    float tolerance, maxStep;         // metres: horizontal joining distance, largest height step
    int minSize;                      // voxels of the smallest patch
  };
  std::vector<DenseSegment> groundDenseTarget(const DenseGroundParams& params = DenseGroundParams(),
                                              std::vector<int>* labels = nullptr);
  std::vector<DenseSegment> segmentDenseTargetAboveGround(float tolerance, int minSize = 1,
                                                          int maxSize = 2147483647, std::vector<int>* labels = nullptr);
  void splitGround(const pcl::PointCloud<pcl::PointXYZI>& cloud, const Twist& pose,
                   pcl::PointCloud<pcl::PointXYZI>& ground, pcl::PointCloud<pcl::PointXYZI>& nonGround,
                   int searchRadius = 1, float maxHeight = 0.1f);

 private:
  typedef pcl::PointCloud<pcl::PointXYZI> Cloud;
  void optimizeTransformTobeMapped();
  void transformAssociateToMap();
  void transformUpdate();
  void pointAssociateToMap(const pcl::PointXYZI& pi, pcl::PointXYZI& po);
  bool createDownsizedMap();

  Time _laserOdometryTime;
  float _scanPeriod;
  const int _stackFrameNum;
  const int _mapFrameNum;
  long _frameCount;
  long _mapFrameCount;
  size_t _maxIterations;
  float _deltaTAbort, _deltaRAbort;

  int _laserCloudCenWidth, _laserCloudCenHeight, _laserCloudCenDepth;
  const size_t _laserCloudWidth, _laserCloudHeight, _laserCloudDepth, _laserCloudNum;

  // clouds in HBM slots: corner last, surf last, full res, corner / surf stack DS, corner / surf from map, surround DS;
  // the 21 x 11 x 21 cube arrays of the reference are two flat point pools on the GPU (see csrc/mappool.cuh)
  b200::DualCloud* _c;
  std::vector<size_t> _laserCloudValidInd, _laserCloudSurroundInd;
  int _mapSizes[4] = {0, 0, 0, 0};

  Twist _transformSum, _transformIncre, _transformTobeMapped, _transformBefMapped, _transformAftMapped;
  std::vector<IMUState2> _imuHistory;

  pcl::VoxelGrid<pcl::PointXYZI> _downSizeFilterCorner, _downSizeFilterSurf, _downSizeFilterMap;
  bool _downsizedMapCreated = false;
  bool _retainFromMap = false;
  float _denseLeaf = 0.f;  // leaf of the whole-run map (0 = never enabled)
  bool _sharded = false;
  int _shardRank = 0, _shardWorld = 1, _shardSlab = 0;  // cube-sharded map (0 = off)

  b200::Context* _gpu;
  b200::GaussNewtonSolver* _solver;
  std::vector<float> _bufA, _bufB;
  size_t _lastIterations = 0;
  double _phase[4] = {0, 0, 0, 0};
};

}  // namespace loam
