// Host side of the laser-mapping drop-in.  Control flow mirrors upstream BasicLaserMapping::process /
// optimizeTransformTobeMapped (src/lib/BasicLaserMapping.cpp:266-599, 626-926): pose prediction, the rolling
// 21 x 11 x 21 grid of 50 m cubes, field-of-view cube selection and map bookkeeping stay here; voxel filters, tree
// builds, the per-iteration correspondence / Jacobian / normal-equation work and the bulk point transforms are GPU
// calls through include/loam_b200.h.
#include "loam_velodyne/BasicLaserMapping.h"

#include <chrono>
#include <cmath>
#include <cstring>
#include <stdexcept>
#include <string>

#include "b200_runtime.h"
#include "host_math.h"
#include "pose_algebra.h"
#include "loam_velodyne/BasicLaserOdometry.h"

namespace loam {

using hostmath::rad2deg;

enum { M_CORNER_LAST = 0, M_SURF_LAST, M_FULL, M_CORNER_STACK_DS, M_SURF_STACK_DS, M_CORNER_FROM_MAP, M_SURF_FROM_MAP,
       M_SURROUND_DS, M_NUM };

BasicLaserMapping::BasicLaserMapping(const float& scanPeriod, const size_t& maxIterations)
    : _scanPeriod(scanPeriod), _stackFrameNum(1), _mapFrameNum(5), _frameCount(0), _mapFrameCount(0),
      _maxIterations(maxIterations), _deltaTAbort(0.05), _deltaRAbort(0.05), _laserCloudCenWidth(10),
      _laserCloudCenHeight(5), _laserCloudCenDepth(10), _laserCloudWidth(21), _laserCloudHeight(11),
      _laserCloudDepth(21), _laserCloudNum(_laserCloudWidth * _laserCloudHeight * _laserCloudDepth),
      _c(new b200::DualCloud[M_NUM]), _gpu(new b200::Context()), _solver(new b200::GaussNewtonSolver()) {
  static const int slots[M_NUM] = {LOAM_B200_C_MAP_CORNER_LAST, LOAM_B200_C_MAP_SURF_LAST, LOAM_B200_C_MAP_FULL,
                                   LOAM_B200_C_MAP_CORNER_STACK_DS, LOAM_B200_C_MAP_SURF_STACK_DS,
                                   LOAM_B200_C_MAP_CORNER_FROM_MAP, LOAM_B200_C_MAP_SURF_FROM_MAP,
                                   LOAM_B200_C_MAP_SURROUND_DS};
  for (int i = 0; i < M_NUM; i++) _c[i].bind(_gpu, slots[i]);
  _frameCount = _stackFrameNum - 1;
  _mapFrameCount = _mapFrameNum - 1;
  _downSizeFilterCorner.setLeafSize(0.2, 0.2, 0.2);
  _downSizeFilterSurf.setLeafSize(0.4, 0.4, 0.4);
}

BasicLaserMapping::~BasicLaserMapping() {
  delete _solver;
  delete[] _c;
  delete _gpu;
}

pcl::PointCloud<pcl::PointXYZI>& BasicLaserMapping::laserCloud() { return _c[M_FULL].hostMutable(); }
pcl::PointCloud<pcl::PointXYZI>& BasicLaserMapping::laserCloudCornerLast() { return _c[M_CORNER_LAST].hostMutable(); }
pcl::PointCloud<pcl::PointXYZI>& BasicLaserMapping::laserCloudSurfLast() { return _c[M_SURF_LAST].hostMutable(); }
pcl::PointCloud<pcl::PointXYZI> const& BasicLaserMapping::laserCloudSurroundDS() const { return _c[M_SURROUND_DS].host(); }
pcl::PointCloud<pcl::PointXYZI> const& BasicLaserMapping::cornerStackDS() const { return _c[M_CORNER_STACK_DS].host(); }
pcl::PointCloud<pcl::PointXYZI> const& BasicLaserMapping::surfStackDS() const { return _c[M_SURF_STACK_DS].host(); }
pcl::PointCloud<pcl::PointXYZI> const& BasicLaserMapping::cornerFromMap() const { return _c[M_CORNER_FROM_MAP].host(); }
pcl::PointCloud<pcl::PointXYZI> const& BasicLaserMapping::surfFromMap() const { return _c[M_SURF_FROM_MAP].host(); }

void BasicLaserMapping::enableSharding(int rank, int world, const unsigned char* ncclId) {
  _sharded = world > 1 && ncclId == nullptr;  // query slices without a communicator: partial sums only (tests)
  if (ncclId)
    _gpu->check(loam_b200_comm_init(_gpu->get(), rank, world, ncclId), "loam_b200_comm_init");
  else
    _gpu->check(loam_b200_map_set_shard(_gpu->get(), rank, world), "loam_b200_map_set_shard");
}

void BasicLaserMapping::exportPeerHandle(unsigned char out64[64]) {
  _gpu->check(loam_b200_peer_export(_gpu->get(), out64), "loam_b200_peer_export");
}

void BasicLaserMapping::enableCubeSharding(int rank, int world, const unsigned char* handles, int slabMetres) {
  _gpu->check(loam_b200_peer_connect(_gpu->get(), rank, world, handles, slabMetres), "loam_b200_peer_connect");
  _sharded = world > 1;  // per-iteration form: the all-reduce is fused into the iteration kernel
  _shardRank = rank;
  _shardWorld = world;
  _shardSlab = slabMetres;
}

void BasicLaserMapping::enableCubeShardingLocal(BasicLaserMapping** objs, int world, int slabMetres) {
  std::vector<loam_b200_ctx*> ctxs((size_t)world);
  for (int r = 0; r < world; r++) ctxs[r] = objs[r]->_gpu->get();
  objs[0]->_gpu->check(loam_b200_peer_connect_local(ctxs.data(), world, slabMetres), "loam_b200_peer_connect_local");
  for (int r = 0; r < world; r++) {
    objs[r]->_sharded = world > 1;
    objs[r]->_shardRank = r;
    objs[r]->_shardWorld = world;
    objs[r]->_shardSlab = slabMetres;
  }
}

void BasicLaserMapping::retainFromMapClouds(bool on) {
  _retainFromMap = on;
  _gpu->check(loam_b200_map_debug_from_map(_gpu->get(), on ? 1 : 0), "loam_b200_map_debug_from_map");
}

void BasicLaserMapping::enableDenseMap(float leaf, long long maxVoxels) {
  _gpu->check(loam_b200_dense_enable(_gpu->get(), leaf, maxVoxels), "loam_b200_dense_enable");
  _denseLeaf = leaf;
}

BasicLaserMapping::DenseMapStats BasicLaserMapping::denseMapStats() {
  long long s[3] = {0, 0, 0};
  _gpu->check(loam_b200_dense_stats(_gpu->get(), s), "loam_b200_dense_stats");
  return DenseMapStats{s[0], s[1], s[2]};
}

void BasicLaserMapping::denseMap(Cloud& out, std::vector<uint32_t>* counts) {
  const int n = (int)denseMapStats().voxels;
  std::vector<float> buf((size_t)n * 4 + 4);
  if (counts) counts->resize((size_t)n);
  int got = 0;
  _gpu->check(loam_b200_dense_export(_gpu->get(), buf.data(), counts && n > 0 ? counts->data() : nullptr, n, &got),
              "loam_b200_dense_export");
  b200::unpack(buf.data(), (size_t)got, out);
}

void BasicLaserMapping::enableDenseVisibility(double hRes, double vRes, double margin) {
  _gpu->check(loam_b200_dense_visibility(_gpu->get(), hRes, vRes, margin), "loam_b200_dense_visibility");
}

void BasicLaserMapping::enableDenseCarving(double margin, double maxRange) {
  _gpu->check(loam_b200_dense_carving(_gpu->get(), margin, maxRange), "loam_b200_dense_carving");
}

void BasicLaserMapping::denseMapFiltered(Cloud& out, double maxMissRatio, std::vector<uint32_t>* counts,
                                         std::vector<uint16_t>* hits, std::vector<uint16_t>* misses) {
  const int n = (int)denseMapStats().voxels;  // the voxels kept are a subset
  std::vector<float> buf((size_t)n * 4 + 4);
  if (counts) counts->resize((size_t)n + 1);
  if (hits) hits->resize((size_t)n + 1);
  if (misses) misses->resize((size_t)n + 1);
  int got = 0;
  _gpu->check(loam_b200_dense_export_filtered(_gpu->get(), maxMissRatio, buf.data(), counts ? counts->data() : nullptr,
                                              hits ? hits->data() : nullptr, misses ? misses->data() : nullptr, n, &got),
              "loam_b200_dense_export_filtered");
  if (counts) counts->resize((size_t)got);
  if (hits) hits->resize((size_t)got);
  if (misses) misses->resize((size_t)got);
  b200::unpack(buf.data(), (size_t)got, out);
}

void BasicLaserMapping::denseMapNormals(pcl::PointCloud<pcl::PointXYZINormal>& out, double maxMissRatio, int radius,
                                        const Vector3& viewpoint, std::vector<uint32_t>* counts) {
  const double vp[3] = {(double)viewpoint.x(), (double)viewpoint.y(), (double)viewpoint.z()};
  denseMapNormals(out, maxMissRatio, radius, vp, counts);
}

void BasicLaserMapping::denseMapNormals(pcl::PointCloud<pcl::PointXYZINormal>& out, double maxMissRatio, int radius,
                                        const double viewpoint[3], std::vector<uint32_t>* counts) {
  const int n = (int)denseMapStats().voxels;  // the voxels kept are a subset
  std::vector<float> buf((size_t)n * 4 + 4), nrm((size_t)n * 4 + 4);
  if (counts) counts->resize((size_t)n + 1);
  int got = 0;
  _gpu->check(loam_b200_dense_export_normals(_gpu->get(), maxMissRatio, radius, viewpoint, buf.data(),
                                             counts ? counts->data() : nullptr, nrm.data(), n, &got),
              "loam_b200_dense_export_normals");
  if (counts) counts->resize((size_t)got);
  out.points.resize((size_t)got);
  bool finite = true;
  for (int i = 0; i < got; i++) {
    pcl::PointXYZINormal& p = out.points[(size_t)i];
    p.x = buf[4 * i + 0];
    p.y = buf[4 * i + 1];
    p.z = buf[4 * i + 2];
    p.intensity = buf[4 * i + 3];
    p.normal_x = nrm[4 * i + 0];
    p.normal_y = nrm[4 * i + 1];
    p.normal_z = nrm[4 * i + 2];
    p.curvature = nrm[4 * i + 3];
    finite = finite && std::isfinite(p.curvature);  // an undefined normal is NaN in all four fields
  }
  out.width = (std::uint32_t)got;
  out.height = 1;
  out.is_dense = finite;
}

size_t BasicLaserMapping::buildDenseTarget(double maxMissRatio, int radius, const Vector3& viewpoint) {
  const double vp[3] = {(double)viewpoint.x(), (double)viewpoint.y(), (double)viewpoint.z()};
  return buildDenseTarget(maxMissRatio, radius, vp);
}

size_t BasicLaserMapping::buildDenseTarget(double maxMissRatio, int radius, const double viewpoint[3]) {
  int n = 0;
  _gpu->check(loam_b200_dense_target_build(_gpu->get(), maxMissRatio, radius, viewpoint, &n),
              "loam_b200_dense_target_build");
  return (size_t)n;
}

void BasicLaserMapping::loadDenseTarget(float leaf, const pcl::PointCloud<pcl::PointXYZINormal>& target) {
  const size_t n = target.points.size();
  std::vector<float> xyzi(n * 4 + 4), nrm(n * 4 + 4);
  for (size_t i = 0; i < n; i++) {
    const pcl::PointXYZINormal& p = target.points[i];
    const float a[4] = {p.x, p.y, p.z, p.intensity}, b[4] = {p.normal_x, p.normal_y, p.normal_z, p.curvature};
    std::memcpy(&xyzi[4 * i], a, sizeof(a));
    std::memcpy(&nrm[4 * i], b, sizeof(b));
  }
  _gpu->check(loam_b200_dense_target_load(_gpu->get(), leaf, xyzi.data(), nrm.data(), (int)n),
              "loam_b200_dense_target_load");
}

size_t BasicLaserMapping::denseTargetSize() {
  int n = 0;
  _gpu->check(loam_b200_dense_target_size(_gpu->get(), &n), "loam_b200_dense_target_size");
  return (size_t)n;
}

// One segmentation of the target through the C ABI: call(labels or nullptr, records, cap, &k) with room for the n
// target voxels' labels and n records (K <= n), the records converted
template <typename F>
static std::vector<BasicLaserMapping::DenseSegment> targetSegments(size_t n, std::vector<int>* labels, F&& call) {
  std::vector<loam_b200_segment> seg(n + 1);
  std::vector<int32_t> lab(labels ? n + 1 : 0);
  const int k = call(labels ? lab.data() : nullptr, seg.data(), (int)n);
  if (labels) labels->assign(lab.begin(), lab.begin() + (ptrdiff_t)n);
  std::vector<BasicLaserMapping::DenseSegment> out((size_t)k);
  for (int i = 0; i < k; i++) {
    const loam_b200_segment& g = seg[(size_t)i];
    BasicLaserMapping::DenseSegment& o = out[(size_t)i];
    o.size = (size_t)g.size;
    o.first = (size_t)g.first;
    for (int a = 0; a < 3; a++) {
      o.lo[a] = g.lo[a];
      o.hi[a] = g.hi[a];
      o.centroid[a] = g.centroid[a];
    }
  }
  return out;
}

std::vector<BasicLaserMapping::DenseSegment> BasicLaserMapping::segmentDenseTarget(float tolerance, int minSize,
                                                                                   int maxSize,
                                                                                   std::vector<int>* labels) {
  return targetSegments(denseTargetSize(), labels, [&](int32_t* lab, loam_b200_segment* seg, int cap) {
    int k = 0;
    _gpu->check(loam_b200_dense_segment(_gpu->get(), tolerance, minSize, maxSize, lab, seg, cap, &k),
                "loam_b200_dense_segment");
    return k;
  });
}

std::vector<BasicLaserMapping::DenseSegment> BasicLaserMapping::groundDenseTarget(const DenseGroundParams& params,
                                                                                  std::vector<int>* labels) {
  const loam_b200_ground_params prm{params.maxSlopeDeg, params.maxCurvature, params.tolerance, params.maxStep,
                                    params.minSize};
  return targetSegments(denseTargetSize(), labels, [&](int32_t* lab, loam_b200_segment* seg, int cap) {
    int k = 0;
    _gpu->check(loam_b200_dense_ground(_gpu->get(), &prm, lab, seg, cap, &k), "loam_b200_dense_ground");
    return k;
  });
}

std::vector<BasicLaserMapping::DenseSegment> BasicLaserMapping::segmentDenseTargetAboveGround(float tolerance,
                                                                                              int minSize, int maxSize,
                                                                                              std::vector<int>* labels) {
  return targetSegments(denseTargetSize(), labels, [&](int32_t* lab, loam_b200_segment* seg, int cap) {
    int k = 0;
    _gpu->check(loam_b200_dense_segment_above_ground(_gpu->get(), tolerance, minSize, maxSize, lab, seg, cap, &k),
                "loam_b200_dense_segment_above_ground");
    return k;
  });
}

void BasicLaserMapping::splitGround(const Cloud& cloud, const Twist& pose, Cloud& ground, Cloud& nonGround,
                                    int searchRadius, float maxHeight) {
  b200::pack(cloud, _bufA);
  loam_b200_pose p;
  b200::fillPose(pose, p);
  const size_t n = cloud.points.size();
  std::vector<int8_t> lab(n + 1);
  int k = 0;
  _gpu->check(loam_b200_dense_ground_cloud(_gpu->get(), _bufA.data(), (int)n, 0, &p, searchRadius, maxHeight,
                                           lab.data(), nullptr, &k),
              "loam_b200_dense_ground_cloud");
  ground.clear();
  nonGround.clear();
  for (size_t i = 0; i < n; i++) {
    if (lab[i] == 1) ground.push_back(cloud.points[i]);
    else if (lab[i] == 0) nonGround.push_back(cloud.points[i]);
  }
}

static Twist twistOf(const float rot[3], const float pos[3]) {
  Twist t;
  t.rot_x = rot[0];
  t.rot_y = rot[1];
  t.rot_z = rot[2];
  t.pos.x() = pos[0];
  t.pos.y() = pos[1];
  t.pos.z() = pos[2];
  return t;
}

static BasicLaserMapping::DenseAlignResult toDenseAlignResult(const loam_b200_align_result& res) {
  BasicLaserMapping::DenseAlignResult out;
  out.pose = twistOf(res.rot, res.pos);
  out.iterations = (size_t)res.iterations;
  out.nSelected = (size_t)res.n_selected;
  out.rms = res.rms;
  out.degenerate = res.degenerate != 0;
  out.converged = res.converged != 0;
  return out;
}

BasicLaserMapping::DenseAlignResult BasicLaserMapping::alignToDenseTarget(const Cloud& cloud, const Twist& initial,
                                                                          int searchRadius, int maxIterations) {
  b200::pack(cloud, _bufA);
  loam_b200_pose pose;
  b200::fillPose(initial, pose);
  loam_b200_align_result res;
  _gpu->check(loam_b200_dense_align(_gpu->get(), _bufA.data(), (int)cloud.points.size(), 0, &pose, searchRadius,
                                    maxIterations, &res),
              "loam_b200_dense_align");
  return toDenseAlignResult(res);
}

static std::vector<loam_b200_pose> posesOf(const std::vector<Twist>& twists) {
  std::vector<loam_b200_pose> p(twists.size());
  for (size_t i = 0; i < twists.size(); i++) b200::fillPose(twists[i], p[i]);
  return p;
}

std::vector<BasicLaserMapping::DenseScore> BasicLaserMapping::scoreDenseTarget(const Cloud& cloud,
                                                                               const std::vector<Twist>& poses,
                                                                               int searchRadius) {
  b200::pack(cloud, _bufA);
  const std::vector<loam_b200_pose> p = posesOf(poses);
  std::vector<int32_t> sel(poses.size() + 1);
  std::vector<float> ss(poses.size() + 1);
  _gpu->check(loam_b200_dense_score(_gpu->get(), _bufA.data(), (int)cloud.points.size(), 0, p.data(), (int)p.size(),
                                    searchRadius, sel.data(), ss.data()),
              "loam_b200_dense_score");
  std::vector<DenseScore> out(poses.size());
  for (size_t i = 0; i < out.size(); i++) out[i] = DenseScore{(size_t)sel[i], ss[i]};
  return out;
}

std::vector<BasicLaserMapping::DenseAlignResult> BasicLaserMapping::alignToDenseTarget(
    const Cloud& cloud, const std::vector<Twist>& initial, int searchRadius, int maxIterations) {
  b200::pack(cloud, _bufA);
  const std::vector<loam_b200_pose> p = posesOf(initial);
  std::vector<loam_b200_align_result> res(initial.size() + 1);
  _gpu->check(loam_b200_dense_align_batch(_gpu->get(), _bufA.data(), (int)cloud.points.size(), 0, p.data(),
                                          (int)p.size(), searchRadius, maxIterations, res.data()),
              "loam_b200_dense_align_batch");
  std::vector<DenseAlignResult> out(initial.size());
  for (size_t i = 0; i < out.size(); i++) out[i] = toDenseAlignResult(res[i]);
  return out;
}

std::vector<BasicLaserMapping::RelocCandidate> BasicLaserMapping::relocalizeInDenseTarget(
    const Cloud& cloud, const std::vector<Twist>& hypotheses, const RelocParams& params, size_t maxCandidates) {
  b200::pack(cloud, _bufA);
  const std::vector<loam_b200_pose> p = posesOf(hypotheses);
  const loam_b200_reloc_params prm{params.scoreRadius, params.coarseRadius, params.fineRadius, params.keep,
                                   params.maxIterations, params.dedupMetres, params.dedupDegrees};
  std::vector<loam_b200_reloc_candidate> res(maxCandidates + 1);
  int n = 0;
  _gpu->check(loam_b200_dense_relocalize(_gpu->get(), _bufA.data(), (int)cloud.points.size(), 0, p.data(),
                                         (int)p.size(), &prm, res.data(), (int)maxCandidates, &n),
              "loam_b200_dense_relocalize");
  std::vector<RelocCandidate> out((size_t)n);
  for (int i = 0; i < n; i++) {
    const loam_b200_reloc_candidate& r = res[(size_t)i];
    out[(size_t)i] = RelocCandidate{(size_t)r.hypothesis, (size_t)r.score_selected, toDenseAlignResult(r.coarse),
                                    toDenseAlignResult(r.fine), (size_t)r.selected, r.rms};
  }
  return out;
}

void BasicLaserMapping::raycastDenseTarget(const Cloud& rays, const Twist& pose, float minRange, float maxRange,
                                           std::vector<float>& range, std::vector<int>* index) {
  b200::pack(rays, _bufA);
  loam_b200_pose p;
  b200::fillPose(pose, p);
  const size_t n = rays.points.size();
  range.resize(n);
  std::vector<int32_t> idx(index ? n : 0);
  _gpu->check(loam_b200_dense_raycast(_gpu->get(), _bufA.data(), (int)n, 0, &p, minRange, maxRange, range.data(),
                                      index ? idx.data() : nullptr),
              "loam_b200_dense_raycast");
  if (index) index->assign(idx.begin(), idx.end());
}

void BasicLaserMapping::buildDenseDistanceField(const int lo[3], const int dims[3], float maxDistance,
                                                std::vector<float>* dist, std::vector<int>* sq) {
  size_t n = 0;
  if (lo && dims && dims[0] > 0 && dims[1] > 0 && dims[2] > 0) n = (size_t)dims[0] * dims[1] * dims[2];
  std::vector<int32_t> s(sq ? n : 0);
  if (dist) dist->resize(n);
  _gpu->check(loam_b200_dense_distance_build(_gpu->get(), lo, dims, maxDistance, dist ? dist->data() : nullptr,
                                             sq ? s.data() : nullptr),
              "loam_b200_dense_distance_build");
  if (sq) sq->assign(s.begin(), s.end());
}

void BasicLaserMapping::queryDenseDistance(const Cloud& points, std::vector<float>& dist, std::vector<float>* grad) {
  b200::pack(points, _bufA);
  const size_t n = points.points.size();
  dist.resize(n);
  if (grad) grad->resize(3 * n);
  _gpu->check(loam_b200_dense_distance_query(_gpu->get(), _bufA.data(), (int)n, 0, dist.data(),
                                             grad ? grad->data() : nullptr),
              "loam_b200_dense_distance_query");
}

static loam_b200_place_params placeParamsOf(const BasicLaserMapping::PlaceParams& p) {
  return loam_b200_place_params{p.rings, p.sectors, p.maxRadius, p.heightOffset, p.minRange, p.maxRange};
}

void BasicLaserMapping::buildDensePlaces(const std::vector<Vector3>& positions, const Cloud& rays,
                                         const PlaceParams& params) {
  b200::pack(rays, _bufA);
  std::vector<float> pos(positions.size() * 3 + 3);
  for (size_t i = 0; i < positions.size(); i++) {
    pos[3 * i] = positions[i].x();
    pos[3 * i + 1] = positions[i].y();
    pos[3 * i + 2] = positions[i].z();
  }
  const loam_b200_place_params prm = placeParamsOf(params);
  _gpu->check(loam_b200_dense_place_build(_gpu->get(), pos.data(), (int)positions.size(), _bufA.data(),
                                          (int)rays.points.size(), &prm),
              "loam_b200_dense_place_build");
}

std::vector<BasicLaserMapping::PlaceMatch> BasicLaserMapping::queryDensePlaces(const Cloud& cloud, size_t topM) {
  b200::pack(cloud, _bufA);
  std::vector<loam_b200_place_match> res(topM + 1);
  int n = 0;
  _gpu->check(loam_b200_dense_place_query(_gpu->get(), _bufA.data(), (int)cloud.points.size(), 0, (int)topM,
                                          res.data(), &n),
              "loam_b200_dense_place_query");
  std::vector<PlaceMatch> out((size_t)n);
  for (int i = 0; i < n; i++) {
    const loam_b200_place_match& r = res[(size_t)i];
    out[(size_t)i] = PlaceMatch{(size_t)r.candidate, r.shift, r.yaw, Vector3(r.pos[0], r.pos[1], r.pos[2]), r.dist};
  }
  return out;
}

std::vector<BasicLaserMapping::RelocCandidate> BasicLaserMapping::relocalizeGlobalInDenseTarget(
    const Cloud& cloud, const GlobalGrid& grid, const RelocParams& params, size_t maxCandidates) {
  b200::pack(cloud, _bufA);
  const loam_b200_reloc_params prm{params.scoreRadius, params.coarseRadius, params.fineRadius, params.keep,
                                   params.maxIterations, params.dedupMetres, params.dedupDegrees};
  std::vector<loam_b200_reloc_candidate> res(maxCandidates + 1);
  int n = 0;
  _gpu->check(loam_b200_dense_relocalize_global(_gpu->get(), _bufA.data(), (int)cloud.points.size(), 0, grid.topM,
                                                grid.yawStepDeg, grid.yawSteps, grid.xzStep, grid.xzSteps, &prm,
                                                res.data(), (int)maxCandidates, &n),
              "loam_b200_dense_relocalize_global");
  std::vector<RelocCandidate> out((size_t)n);
  for (int i = 0; i < n; i++) {
    const loam_b200_reloc_candidate& r = res[(size_t)i];
    out[(size_t)i] = RelocCandidate{(size_t)r.hypothesis, (size_t)r.score_selected, toDenseAlignResult(r.coarse),
                                    toDenseAlignResult(r.fine), (size_t)r.selected, r.rms};
  }
  return out;
}

std::vector<Twist> BasicLaserMapping::relocalizationGrid(const Twist& prior, float yawStepDeg, int yawSteps,
                                                         float xzStep, int xzSteps) {
  loam_b200_pose p;
  b200::fillPose(prior, p);
  int n = 0;
  int rc = loam_b200_reloc_grid(&p, yawStepDeg, yawSteps, xzStep, xzSteps, nullptr, 0, &n);
  std::vector<loam_b200_pose> grid;
  if (rc == LOAM_B200_ERR_CAPACITY) {
    grid.resize((size_t)n);
    rc = loam_b200_reloc_grid(&p, yawStepDeg, yawSteps, xzStep, xzSteps, grid.data(), n, &n);
  }
  if (rc != LOAM_B200_OK)
    throw std::runtime_error(std::string("loam_b200_reloc_grid: ") + loam_b200_strerror(rc));
  std::vector<Twist> out((size_t)n);
  for (int i = 0; i < n; i++) out[(size_t)i] = twistOf(grid[(size_t)i].rot, grid[(size_t)i].pos);
  return out;
}

long long BasicLaserMapping::denseTableSlots() {
  long long n = 0;
  _gpu->check(loam_b200_debug_dense_table_slots(_gpu->get(), &n), "loam_b200_debug_dense_table_slots");
  return n;
}

void BasicLaserMapping::denseMapSnapshot(DenseMapSnapshot& out) {
  const int n = (int)denseMapStats().voxels;
  out.leaf = _denseLeaf;
  out.keys.resize((size_t)n + 1);
  out.counts.resize((size_t)n + 1);
  out.hits.resize((size_t)n + 1);
  out.misses.resize((size_t)n + 1);
  out.sums.resize(4 * ((size_t)n + 1));
  int got = 0;
  _gpu->check(loam_b200_dense_snapshot(_gpu->get(), out.keys.data(), out.counts.data(), out.hits.data(),
                                       out.misses.data(), out.sums.data(), n, &got),
              "loam_b200_dense_snapshot");
  out.keys.resize((size_t)got);
  out.counts.resize((size_t)got);
  out.hits.resize((size_t)got);
  out.misses.resize((size_t)got);
  out.sums.resize(4 * (size_t)got);
}

void BasicLaserMapping::mergeDenseMap(const DenseMapSnapshot& snap, const Twist* pose) {
  const size_t n = snap.counts.size();
  if (snap.hits.size() != n || snap.misses.size() != n || snap.sums.size() != 4 * n)
    throw std::invalid_argument("BasicLaserMapping::mergeDenseMap: the snapshot's arrays differ in length");
  loam_b200_pose p;
  if (pose) b200::fillPose(*pose, p);
  _gpu->check(loam_b200_dense_merge(_gpu->get(), snap.counts.data(), snap.hits.data(), snap.misses.data(),
                                    snap.sums.data(), (int)n, pose ? &p : nullptr),
              "loam_b200_dense_merge");
}

void BasicLaserMapping::clearDenseMap() {
  _gpu->check(loam_b200_dense_clear(_gpu->get()), "loam_b200_dense_clear");
}

void BasicLaserMapping::adopt(BasicLaserOdometry& odom) {
  static const int to[3] = {M_CORNER_LAST, M_SURF_LAST, M_FULL};
  int dstSlots[3], srcSlots[3];
  for (int i = 0; i < 3; i++) {
    b200::DualCloud& src = odom.deviceCloud(i);
    src.ensureDevice();
    dstSlots[i] = _c[to[i]].slot();
    srcSlots[i] = src.slot();
  }
  _gpu->check(loam_b200_cloud_copy_many(_gpu->get(), dstSlots, odom.deviceContext()->get(), srcSlots, 3),
              "loam_b200_cloud_copy_many");
  for (int i = 0; i < 3; i++) _c[to[i]].deviceWritten((int)odom.deviceCloud(i).size());
  updateOdometry(odom.transformSum());
}

// Pose prediction: compose (Sum, BefMapped, AftMapped) into TobeMapped, closed-form ZXY Euler algebra as published
// with LOAM (upstream :103-167).
void BasicLaserMapping::transformAssociateToMap() {
  hostmath::associateToMap(_transformSum, _transformBefMapped, _transformAftMapped, _transformIncre, _transformTobeMapped);
}

void BasicLaserMapping::transformUpdate() {
  if (!_imuHistory.empty()) {
    size_t imuIdx = 0;
    while (imuIdx < _imuHistory.size() - 1 && toSec(_laserOdometryTime - _imuHistory[imuIdx].stamp) + _scanPeriod > 0)
      imuIdx++;
    IMUState2 imuCur;
    if (imuIdx == 0 || toSec(_laserOdometryTime - _imuHistory[imuIdx].stamp) + _scanPeriod > 0) {
      imuCur = _imuHistory[imuIdx];
    } else {
      const float ratio = (float)((toSec(_imuHistory[imuIdx].stamp - _laserOdometryTime) - _scanPeriod) /
                                  toSec(_imuHistory[imuIdx].stamp - _imuHistory[imuIdx - 1].stamp));
      IMUState2::interpolate(_imuHistory[imuIdx], _imuHistory[imuIdx - 1], ratio, imuCur);
    }
    _transformTobeMapped.rot_x = 0.998 * _transformTobeMapped.rot_x.rad() + 0.002 * imuCur.pitch.rad();
    _transformTobeMapped.rot_z = 0.998 * _transformTobeMapped.rot_z.rad() + 0.002 * imuCur.roll.rad();
  }
  _transformBefMapped = _transformSum;
  _transformAftMapped = _transformTobeMapped;
}

void BasicLaserMapping::pointAssociateToMap(const pcl::PointXYZI& pi, pcl::PointXYZI& po) {
  po.x = pi.x;
  po.y = pi.y;
  po.z = pi.z;
  po.intensity = pi.intensity;
  hostmath::rotateZXY(po, _transformTobeMapped.rot_z, _transformTobeMapped.rot_x, _transformTobeMapped.rot_y);
  po.x += _transformTobeMapped.pos.x();
  po.y += _transformTobeMapped.pos.y();
  po.z += _transformTobeMapped.pos.z();
}

bool BasicLaserMapping::createDownsizedMap() {
  _mapFrameCount++;
  if (_mapFrameCount < _mapFrameNum) return false;
  _mapFrameCount = 0;
  // corner + surface points of the 5 x 5 x 5 surround cubes, filtered with the CORNER filter (upstream :251-262;
  // _downSizeFilterMap is configurable but never used there either)
  std::vector<int32_t> cubes(_laserCloudSurroundInd.begin(), _laserCloudSurroundInd.end());
  const int cen[3] = {_laserCloudCenWidth, _laserCloudCenHeight, _laserCloudCenDepth};
  // computed asynchronously on an auxiliary context (it is a visualisation product and costs half a sweep); the
  // accessor laserCloudSurroundDS() waits for it
  _gpu->check(loam_b200_map_surround_async(_gpu->get(), cen, cubes.data(), (int)cubes.size(),
                                           b200::leafOf(_downSizeFilterCorner)),
              "loam_b200_map_surround_async");
  _c[M_SURROUND_DS].deviceWrittenLazy();
  return true;
}

bool BasicLaserMapping::process(Time const& laserOdometryTime) {
  _frameCount++;
  if (_frameCount < _stackFrameNum) return false;
  _frameCount = 0;
  _laserOdometryTime = laserOdometryTime;

  transformAssociateToMap();

  pcl::PointXYZI pointOnYAxis;
  pointOnYAxis.x = 0.0;
  pointOnYAxis.y = 10.0;
  pointOnYAxis.z = 0.0;
  pointAssociateToMap(pointOnYAxis, pointOnYAxis);

  const double CUBE_SIZE = 50.0, CUBE_HALF = CUBE_SIZE / 2;
  int centerCubeI = int((_transformTobeMapped.pos.x() + CUBE_HALF) / CUBE_SIZE) + _laserCloudCenWidth;
  int centerCubeJ = int((_transformTobeMapped.pos.y() + CUBE_HALF) / CUBE_SIZE) + _laserCloudCenHeight;
  int centerCubeK = int((_transformTobeMapped.pos.z() + CUBE_HALF) / CUBE_SIZE) + _laserCloudCenDepth;
  if (_transformTobeMapped.pos.x() + CUBE_HALF < 0) centerCubeI--;
  if (_transformTobeMapped.pos.y() + CUBE_HALF < 0) centerCubeJ--;
  if (_transformTobeMapped.pos.z() + CUBE_HALF < 0) centerCubeK--;

  // Rolling the grid (upstream :311-441 moves cube pointers and clears the slab that wraps around): with the flat
  // GPU pools a point's cube follows from its position and these centre offsets, so only the offsets move; points
  // whose cube leaves the grid are dropped by the next end-of-sweep pass.
  while (centerCubeI < 3) { centerCubeI++; _laserCloudCenWidth++; }
  while (centerCubeI >= (int)_laserCloudWidth - 3) { centerCubeI--; _laserCloudCenWidth--; }
  while (centerCubeJ < 3) { centerCubeJ++; _laserCloudCenHeight++; }
  while (centerCubeJ >= (int)_laserCloudHeight - 3) { centerCubeJ--; _laserCloudCenHeight--; }
  while (centerCubeK < 3) { centerCubeK++; _laserCloudCenDepth++; }
  while (centerCubeK >= (int)_laserCloudDepth - 3) { centerCubeK--; _laserCloudCenDepth--; }

  // 5 x 5 x 5 neighbourhood; a cube is "valid" when one of its corners lies within 30..150 degrees of the sensor's
  // up axis (law-of-cosines test against a point 10 m up the y axis, upstream :456-489)
  _laserCloudValidInd.clear();
  _laserCloudSurroundInd.clear();
  const pcl::PointXYZI sensorPos = (pcl::PointXYZI)_transformTobeMapped.pos;
  for (int i = centerCubeI - 2; i <= centerCubeI + 2; i++) {
    for (int j = centerCubeJ - 2; j <= centerCubeJ + 2; j++) {
      for (int k = centerCubeK - 2; k <= centerCubeK + 2; k++) {
        if (i < 0 || i >= (int)_laserCloudWidth || j < 0 || j >= (int)_laserCloudHeight || k < 0 ||
            k >= (int)_laserCloudDepth)
          continue;
        const float centerX = 50.0f * (i - _laserCloudCenWidth);
        const float centerY = 50.0f * (j - _laserCloudCenHeight);
        const float centerZ = 50.0f * (k - _laserCloudCenDepth);
        bool isInLaserFOV = false;
        for (int ii = -1; ii <= 1; ii += 2) {
          for (int jj = -1; jj <= 1; jj += 2) {
            for (int kk = -1; kk <= 1; kk += 2) {
              const float cx = centerX + 25.0f * ii, cy = centerY + 25.0f * jj, cz = centerZ + 25.0f * kk;
              const float d1x = sensorPos.x - cx, d1y = sensorPos.y - cy, d1z = sensorPos.z - cz;
              const float squaredSide1 = d1x * d1x + d1y * d1y + d1z * d1z;
              const float d2x = pointOnYAxis.x - cx, d2y = pointOnYAxis.y - cy, d2z = pointOnYAxis.z - cz;
              const float squaredSide2 = d2x * d2x + d2y * d2y + d2z * d2z;
              const float check1 = 100.0f + squaredSide1 - squaredSide2 - 10.0f * std::sqrt(3.0f) * std::sqrt(squaredSide1);
              const float check2 = 100.0f + squaredSide1 - squaredSide2 + 10.0f * std::sqrt(3.0f) * std::sqrt(squaredSide1);
              if (check1 < 0 && check2 > 0) isInLaserFOV = true;
            }
          }
        }
        const size_t cubeIdx = i + _laserCloudWidth * j + _laserCloudWidth * _laserCloudHeight * k;
        if (isInLaserFOV) _laserCloudValidInd.push_back(cubeIdx);
        _laserCloudSurroundInd.push_back(cubeIdx);
      }
    }
  }

  // GPU: feature stacks (to map and back with the predicted pose, voxel filters), surrounding-map clouds of the valid
  // cubes and their BVHs (upstream :282-292, :503-527, :636-637)
  _c[M_CORNER_LAST].ensureDevice();
  _c[M_SURF_LAST].ensureDevice();
  _c[M_FULL].ensureDevice();
  std::vector<int32_t> valid(_laserCloudValidInd.begin(), _laserCloudValidInd.end());
  loam_b200_map_window win;
  win.cen[0] = _laserCloudCenWidth;
  win.cen[1] = _laserCloudCenHeight;
  win.cen[2] = _laserCloudCenDepth;
  win.valid_cubes = valid.data();
  win.n_valid = (int)valid.size();
  win.corner_leaf = b200::leafOf(_downSizeFilterCorner);
  win.surf_leaf = b200::leafOf(_downSizeFilterSurf);
  auto now = [] { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); };
  const double tp0 = now();
  loam_b200_pose predicted;
  b200::fillPose(_transformTobeMapped, predicted);
  _gpu->check(loam_b200_map_begin_sweep(_gpu->get(), &predicted, &win, _mapSizes), "loam_b200_map_begin_sweep");
  // the persistent GPU map only reports how many points the cubes in view hold; the clouds themselves are
  // materialised on request (retainFromMapClouds)
  _c[M_CORNER_FROM_MAP].deviceWritten(_retainFromMap ? _mapSizes[0] : 0);
  _c[M_SURF_FROM_MAP].deviceWritten(_retainFromMap ? _mapSizes[1] : 0);
  _c[M_CORNER_STACK_DS].deviceWritten(_mapSizes[2]);
  _c[M_SURF_STACK_DS].deviceWritten(_mapSizes[3]);

  const double tp1 = now();
  optimizeTransformTobeMapped();
  const double tp2 = now();

  // GPU: insert the down-sized stack points with the optimised pose, voxel-filter every valid cube, move the
  // full-resolution cloud into the map frame (upstream :536-595)
  loam_b200_pose optimised;
  b200::fillPose(_transformTobeMapped, optimised);
  // issued by the context's helper thread: nothing below depends on it, the next call on the context joins it
  _gpu->check(loam_b200_map_end_sweep_async(_gpu->get(), &optimised), "loam_b200_map_end_sweep_async");
  _c[M_FULL].deviceWritten((int)_c[M_FULL].size());
  const double tp3 = now();

  _downsizedMapCreated = createDownsizedMap();
  const double tp4 = now();
  _phase[0] = tp1 - tp0; _phase[1] = tp2 - tp1; _phase[2] = tp3 - tp2; _phase[3] = tp4 - tp3;
  return true;
}

void BasicLaserMapping::updateIMU(IMUState2 const& newState) {
  _imuHistory.push_back(newState);
  if (_imuHistory.size() > 200) _imuHistory.erase(_imuHistory.begin());
}

void BasicLaserMapping::updateOdometry(double pitch, double yaw, double roll, double x, double y, double z) {
  _transformSum.rot_x = pitch;
  _transformSum.rot_y = yaw;
  _transformSum.rot_z = roll;
  _transformSum.pos.x() = float(x);
  _transformSum.pos.y() = float(y);
  _transformSum.pos.z() = float(z);
}

void BasicLaserMapping::updateOdometry(Twist const& twist) { _transformSum = twist; }

void BasicLaserMapping::optimizeTransformTobeMapped() {
  _lastIterations = 0;
  _solver->isDegenerate = false;  // a local of optimizeTransformTobeMapped() upstream (:640): fresh every sweep
  // _laserCloudCornerFromMap->size() <= 10 || _laserCloudSurfFromMap->size() <= 100 (upstream :628-629); the trees
  // and the query stacks were prepared by loam_b200_map_begin_sweep
  if (_mapSizes[0] <= 10 || _mapSizes[1] <= 100) return;

  if (!_sharded && b200::deviceResidentLoops()) {
    // optional: the whole iteration loop (:646-922) on the device (loam_b200_map_solve; with a communicator the all-reduce of the
    // partial normal equations sits between the iteration kernel and the step kernel); the per-iteration form below
    // remains for query slices without a communicator
    const float rot[3] = {_transformTobeMapped.rot_x.rad(), _transformTobeMapped.rot_y.rad(), _transformTobeMapped.rot_z.rad()};
    const float pos[3] = {_transformTobeMapped.pos.x(), _transformTobeMapped.pos.y(), _transformTobeMapped.pos.z()};
    loam_b200_lm_result res;
    _gpu->check(loam_b200_map_solve(_gpu->get(), rot, pos, (int)_maxIterations, _deltaTAbort, _deltaRAbort, &res),
                "loam_b200_map_solve");
    _lastIterations = (size_t)res.iterations;
    _transformTobeMapped.rot_x = res.rot[0];
    _transformTobeMapped.rot_y = res.rot[1];
    _transformTobeMapped.rot_z = res.rot[2];
    _transformTobeMapped.pos.x() = res.pos[0];
    _transformTobeMapped.pos.y() = res.pos[1];
    _transformTobeMapped.pos.z() = res.pos[2];
    transformUpdate();
    return;
  }
  for (size_t iterCount = 0; iterCount < _maxIterations; iterCount++) {
    _lastIterations = iterCount + 1;
    loam_b200_pose pose;
    b200::fillPose(_transformTobeMapped, pose);
    loam_b200_normal_eq ne;
    _gpu->check(loam_b200_map_iterate(_gpu->get(), &pose, &ne), "loam_b200_map_iterate");
    if (ne.n_selected < 50) continue;

    float x[6];
    _solver->solve(ne, iterCount == 0, 100.f, x);

    _transformTobeMapped.rot_x += x[0];
    _transformTobeMapped.rot_y += x[1];
    _transformTobeMapped.rot_z += x[2];
    _transformTobeMapped.pos.x() += x[3];
    _transformTobeMapped.pos.y() += x[4];
    _transformTobeMapped.pos.z() += x[5];

    const float deltaR = std::sqrt(std::pow(rad2deg(x[0]), 2) + std::pow(rad2deg(x[1]), 2) + std::pow(rad2deg(x[2]), 2));
    const float deltaT = std::sqrt(std::pow(x[3] * 100, 2) + std::pow(x[4] * 100, 2) + std::pow(x[5] * 100, 2));
    if (deltaR < _deltaRAbort && deltaT < _deltaTAbort) break;
  }
  transformUpdate();
}

void BasicLaserMapping::seedMap(Cloud const& cornerPoints, Cloud const& surfPoints) {
  // points outside the 21 x 11 x 21 grid are dropped by the first end-of-sweep pass, like upstream's insertion
  // (:548-554) would never have stored them
  const Cloud* in[2] = {&cornerPoints, &surfPoints};
  for (int kind = 0; kind < 2; kind++) {
    if (_shardSlab > 0 && _shardWorld > 1) {
      // cube-sharded map: this rank only holds the points of the slabs it owns and their halo (start-up, not hot path)
      _bufA.clear();
      _bufA.reserve(in[kind]->points.size() * 4 / _shardWorld + 64);
      for (auto const& p : in[kind]->points)
        if (loam_b200_shard_stores(p.x, _shardRank, _shardWorld, _shardSlab) == 1) {
          _bufA.push_back(p.x); _bufA.push_back(p.y); _bufA.push_back(p.z); _bufA.push_back(p.intensity);
        }
    } else {
      b200::pack(*in[kind], _bufA);
    }
    _gpu->check(loam_b200_map_pool_append(_gpu->get(), kind, _bufA.data(), (int)(_bufA.size() / 4)), "loam_b200_map_pool_append");
  }
}

void BasicLaserMapping::collectMap(Cloud& corner, Cloud& surf) const {
  Cloud* out[2] = {&corner, &surf};
  const int slot[2] = {LOAM_B200_C_MAP_CORNER_POOL, LOAM_B200_C_MAP_SURF_POOL};
  std::vector<float> buf;
  for (int k = 0; k < 2; k++) {
    const int n = _gpu->created() ? loam_b200_cloud_size(_gpu->get(), slot[k]) : 0;
    buf.resize((size_t)n * 4 + 4);
    int got = 0;
    if (n > 0) _gpu->check(loam_b200_cloud_download(_gpu->get(), slot[k], buf.data(), n, &got), "loam_b200_cloud_download");
    b200::unpack(buf.data(), (size_t)got, *out[k]);
  }
}

}  // namespace loam
