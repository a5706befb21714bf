// C handles over the C++ drop-in classes (include/loam_b200_host.h).
#include "loam_b200_host.h"

#include <chrono>
#include <condition_variable>
#include <cstring>
#include <deque>
#include <exception>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include "b200_runtime.h"
#include "loam_velodyne/BasicLaserMapping.h"
#include "loam_velodyne/BasicLaserOdometry.h"
#include "loam_velodyne/BasicScanRegistration.h"
#include "loam_velodyne/BasicTransformMaintenance.h"

namespace {

namespace b200 = loam::b200;
typedef pcl::PointCloud<pcl::PointXYZI> Cloud;
thread_local std::string g_err;

template <typename F>
int guarded(F&& f) {
  try {
    return f();
  } catch (const std::exception& e) {
    g_err = e.what();
    return -1;
  } catch (...) {
    g_err = "unknown exception";
    return -1;
  }
}

void fill(Cloud& c, const float* p, int n) {
  loam::b200::unpack(p, (size_t)(n > 0 ? n : 0), c);
}
void dump(const Cloud& c, float* out) {
  for (size_t i = 0; i < c.points.size(); i++) {
    out[4 * i + 0] = c.points[i].x;
    out[4 * i + 1] = c.points[i].y;
    out[4 * i + 2] = c.points[i].z;
    out[4 * i + 3] = c.points[i].intensity;
  }
}
void twist6(const loam::Twist& t, float* o) {
  o[0] = t.rot_x.rad(); o[1] = t.rot_y.rad(); o[2] = t.rot_z.rad();
  o[3] = t.pos.x(); o[4] = t.pos.y(); o[5] = t.pos.z();
}
double now() { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); }

struct RegH {
  loam::BasicScanRegistration r;
  std::vector<Cloud> rings;
  const Cloud& cloud(int which) {
    switch (which) {
      case 0: return r.laserCloud();
      case 1: return r.cornerPointsSharp();
      case 2: return r.cornerPointsLessSharp();
      case 3: return r.surfacePointsFlat();
      default: return r.surfacePointsLessFlat();
    }
  }
  const std::vector<int>& index(int which) {
    return which == 1 ? r.sharpIndices() : which == 2 ? r.lessSharpIndices() : r.flatIndices();
  }
  // the reference entry point: one pcl cloud per ring (BasicScanRegistration.h:142)
  void process(const float* pts, const int* ring_sizes, int n_rings) {
    rings.resize(n_rings);
    int off = 0;
    for (int i = 0; i < n_rings; i++) {
      fill(rings[i], pts + 4 * (size_t)off, ring_sizes[i]);
      off += ring_sizes[i];
    }
    r.processScanlines(loam::Time(), rings);
  }
};
struct OdomH {
  loam::BasicLaserOdometry o;
  OdomH(float sp, int it) : o(sp, it) {}
  const Cloud& cloud(int which) {
    return which == 0 ? *o.lastCornerCloud() : which == 1 ? *o.lastSurfaceCloud() : o.deviceCloud(2).host();
  }
};
struct StreamRunner;
struct MapH {
  loam::BasicLaserMapping m;
  Cloud scratchA, scratchB;
  StreamRunner* runner = nullptr;  // the pipeline's stage threads when this is a streaming pipeline's mapping object
  MapH(float sp, int it) : m(sp, it) {}
  const Cloud& cloud(int which) {
    switch (which) {
      case 0: return m.laserCloud();
      case 1: return m.laserCloudSurroundDS();
      case 2: return m.cornerFromMap();
      case 3: return m.surfFromMap();
      case 4: return m.cornerStackDS();
      case 5: return m.surfStackDS();
      case 6: m.collectMap(scratchA, scratchB); return scratchA;
      default: m.collectMap(scratchA, scratchB); return scratchB;
    }
  }
};
struct PipeH {
  RegH reg;
  OdomH odom;
  MapH map;
  StreamRunner* runner = nullptr;
  PipeH(float sp, int oi, int mi) : odom(sp, oi), map(sp, mi) {}
  ~PipeH();
};

// ---- the three stages as three concurrent single-threaded workers over consecutive sweeps ------------------------------
// This is how the reference is deployed: multiScanRegistration, laserOdometry and laserMapping are separate single-
// threaded ROS nodes (CMakeLists.txt:40-50), so while laserMapping works on sweep k, laserOdometry works on k + 1 and the
// registration on k + 2.  Here each stage object has its own context / stream and one host thread; the ROS topics between
// the nodes (ScanRegistration.cpp:187-199, LaserOdometry.cpp:286-330) are the device-to-device adopt() hand-offs, taken by
// the consumer while the producer waits (a stage's output clouds are overwritten by its next sweep).  Results are the
// same as the sequential chain, bit for bit: every stage still sees the sweeps in order and only through the hand-offs.
struct SweepJob {
  const float* pts;
  const void* d_pts;
  std::vector<int> rings;
  long id;
};
struct SweepResult {
  long id;
  int ok;
  float odom[6], aft[6];
};

struct StreamRunner {
  PipeH* p;
  int device;
  std::thread th[3];
  std::mutex m;
  std::condition_variable cv;
  std::deque<SweepJob> in;
  std::deque<SweepResult> out;
  long next_id = 0, reg_done = 0, odom_done = 0, n_submitted = 0, n_finished = 0, n_collected = 0;
  bool reg_ready = false, odom_ready = false, stop = false;
  std::string err;
  // seconds each stage spent working / waiting for its neighbours (loam_b200_pipeline_stage_seconds)
  double busy[3] = {0, 0, 0}, idle[3] = {0, 0, 0}, handoff[3] = {0, 0, 0};
  double t_reset = 0.0;  // waiting that began before the last reset of the counters is not counted
  static constexpr size_t MAX_QUEUED = 2;

  explicit StreamRunner(PipeH* pipe) : p(pipe), device(loam::b200::defaultDevice()) {
    // users of the streaming form synchronise through loam_b200_pipeline_sync: the helper thread may record its sequence
    auto* mc = p->map.m.deviceContext();
    mc->check(loam_b200_allow_async_capture(mc->get(), 1), "loam_b200_allow_async_capture");
    th[0] = std::thread([this] { run(0); });
    th[1] = std::thread([this] { run(1); });
    th[2] = std::thread([this] { run(2); });
  }
  ~StreamRunner() {
    {
      std::lock_guard<std::mutex> lk(m);
      stop = true;
    }
    cv.notify_all();
    for (auto& t : th)
      if (t.joinable()) t.join();
  }
  // Stage hand-offs are latency critical (the cycle of the pipeline is odometry + both hand-offs): poll the condition for
  // a short while before falling back to the condition variable (a futex wake-up costs 10-50 us on a busy box).
  template <typename PRED>
  void wait_for(std::unique_lock<std::mutex>& lk, PRED pred) {
    if (pred()) return;
    const auto t0 = std::chrono::steady_clock::now();
    for (;;) {
      lk.unlock();
      for (int i = 0; i < 64; i++) {
#if defined(__x86_64__)
        __builtin_ia32_pause();
#endif
      }
      lk.lock();
      if (pred()) return;
      if (std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count() > 300e-6) break;
    }
    cv.wait(lk, pred);
  }
  void fail(const char* what) {
    std::lock_guard<std::mutex> lk(m);
    if (err.empty()) err = what;
    stop = true;
    cv.notify_all();
  }
  void run(int stage) {
    loam_b200_bind_thread(device);
    try {
      if (stage == 0) stage_reg(); else if (stage == 1) stage_odom(); else stage_map();
    } catch (const std::exception& e) {
      fail(e.what());
    } catch (...) {
      fail("unknown exception in a pipeline stage");
    }
  }
  void stage_reg() {
    for (;;) {
      SweepJob job;
      const double tw = now();
      {
        std::unique_lock<std::mutex> lk(m);
        // the previous sweep's clouds must have been taken over before they are overwritten
        wait_for(lk, [this] { return stop || (!in.empty() && !reg_ready); });
        if (stop) return;
        job = std::move(in.front());
        in.pop_front();
      }
      cv.notify_all();
      const double tb = now();
      if (job.d_pts)
        p->reg.r.processDeviceSweep(loam::Time(), job.d_pts, job.rings.data(), (int)job.rings.size());
      else
        p->reg.r.processPackedSweep(loam::Time(), job.pts, job.rings.data(), (int)job.rings.size());
      idle[0] += tb - std::max(tw, t_reset);
      busy[0] += now() - tb;
      {
        std::lock_guard<std::mutex> lk(m);
        reg_ready = true;
      }
      cv.notify_all();
    }
  }
  void stage_odom() {
    auto& o = p->odom.o;
    for (;;) {
      const double tw = now();
      {
        std::unique_lock<std::mutex> lk(m);
        // adopt() overwrites the full-resolution cloud the mapping stage takes from this object
        wait_for(lk, [this] { return stop || (reg_ready && !odom_ready); });
        if (stop) return;
      }
      const double ta = now();
      o.adopt(p->reg.r);  // the registration thread is parked until reg_ready drops
      {
        std::lock_guard<std::mutex> lk(m);
        reg_ready = false;
      }
      cv.notify_all();
      const double tb = now();
      o.process();
      o.transformLaserCloudToEnd();
      idle[1] += ta - std::max(tw, t_reset);
      handoff[1] += tb - ta;
      busy[1] += now() - tb;
      {
        std::lock_guard<std::mutex> lk(m);
        odom_ready = true;
      }
      cv.notify_all();
    }
  }
  void stage_map() {
    auto& o = p->odom.o;
    auto& mp = p->map.m;
    for (;;) {
      const double tw = now();
      {
        std::unique_lock<std::mutex> lk(m);
        wait_for(lk, [this] { return stop || odom_ready; });
        if (stop) return;
      }
      const double ta = now();
      SweepResult r;
      mp.adopt(o);  // the odometry thread is parked until odom_ready drops
      twist6(o.transformSum(), r.odom);
      {
        std::lock_guard<std::mutex> lk(m);
        odom_ready = false;
      }
      cv.notify_all();
      const double tb = now();
      r.ok = mp.process(loam::Time()) ? 1 : 0;
      twist6(mp.transformAftMapped(), r.aft);
      idle[2] += ta - std::max(tw, t_reset);
      handoff[2] += tb - ta;
      busy[2] += now() - tb;
      {
        std::lock_guard<std::mutex> lk(m);
        r.id = n_finished++;
        out.push_back(r);
      }
      cv.notify_all();
    }
  }
  int submit(const float* pts, const void* d_pts, const int* rings, int n_rings) {
    SweepJob job{pts, d_pts, std::vector<int>(rings, rings + n_rings), 0};
    std::unique_lock<std::mutex> lk(m);
    cv.wait(lk, [this] { return stop || in.size() < MAX_QUEUED; });
    if (stop) { g_err = err.empty() ? "pipeline stopped" : err; return -1; }
    job.id = n_submitted++;
    in.push_back(std::move(job));
    lk.unlock();
    cv.notify_all();
    return 0;
  }
  // a sweep is in flight from its submit() until its result has been collected
  bool in_flight() {
    std::lock_guard<std::mutex> lk(m);
    return n_collected != n_submitted;
  }
  // 1 = a result was returned, 0 = none pending / none ready (wait == 0), -1 = a stage failed
  int collect(int wait, SweepResult* r) {
    std::unique_lock<std::mutex> lk(m);
    if (wait) cv.wait(lk, [this] { return stop || !out.empty() || n_finished == n_submitted; });
    if (!out.empty()) {
      *r = out.front();
      out.pop_front();
      n_collected++;
      return 1;
    }
    if (!err.empty()) { g_err = err; return -1; }
    return 0;
  }
};

PipeH::~PipeH() { delete runner; }

// the mapping object of a streaming pipeline belongs to its stage thread while sweeps are in flight
int map_in_flight(MapH* h) {
  if (!h->runner || !h->runner->in_flight()) return 0;
  g_err = "the pipeline has sweeps in flight (submitted, result not collected yet): collect them first";
  return LOAM_B200_ERR_STATE;
}

}  // namespace

extern "C" {

const char* loam_b200_host_last_error(void) { return g_err.c_str(); }
void loam_b200_host_set_device(int device) { loam::b200::setDefaultDevice(device); }

int loam_b200_host_gn_solve(const float* AtA, const float* AtB, int first_iteration, float eigen_threshold, float* x_out6,
                            int* degenerate_out) {
  if (!AtA || !AtB || !x_out6) return -1;
  loam_b200_normal_eq ne;
  std::memset(&ne, 0, sizeof ne);
  std::memcpy(ne.AtA, AtA, sizeof ne.AtA);
  std::memcpy(ne.AtB, AtB, sizeof ne.AtB);
  loam::b200::GaussNewtonSolver solver;
  solver.solve(ne, first_iteration != 0, eigen_threshold, x_out6);
  if (degenerate_out) *degenerate_out = solver.isDegenerate ? 1 : 0;
  return 0;
}

int loam_b200_transform_maintenance(const float* sum6, const float* bef6, const float* aft6, float* mapped_out6) {
  if (!sum6 || !bef6 || !aft6 || !mapped_out6) return -1;
  loam::BasicTransformMaintenance tm;
  tm.updateOdometry(sum6[0], sum6[1], sum6[2], sum6[3], sum6[4], sum6[5]);
  tm.updateMappingTransform(aft6[0], aft6[1], aft6[2], aft6[3], aft6[4], aft6[5], bef6[0], bef6[1], bef6[2], bef6[3], bef6[4],
                            bef6[5]);
  tm.transformAssociateToMap();
  for (int i = 0; i < 6; i++) mapped_out6[i] = tm.transformMapped()[i];
  return 0;
}

void* loam_b200_scanreg_create(void) { return new RegH(); }
void loam_b200_scanreg_destroy(void* h) { delete (RegH*)h; }
int loam_b200_scanreg_configure(void* h, float scanPeriod, int nFeatureRegions, int curvatureRegion, int maxCornerSharp,
                                int maxSurfaceFlat, float lessFlatFilterSize, float surfaceCurvatureThreshold) {
  return guarded([&] {
    loam::RegistrationParams p(scanPeriod, 200, nFeatureRegions, curvatureRegion, maxCornerSharp, maxSurfaceFlat,
                               lessFlatFilterSize, surfaceCurvatureThreshold);
    return ((RegH*)h)->r.configure(p) ? 0 : -1;
  });
}
int loam_b200_scanreg_process(void* h, const float* pts, const int* ring_sizes, int n_rings) {
  return guarded([&] { ((RegH*)h)->process(pts, ring_sizes, n_rings); return 0; });
}
int loam_b200_scanreg_process_unordered(void* h, const float* xyz, int n, float lower_bound_deg, float upper_bound_deg,
                                        int n_rings) {
  return guarded([&] {
    ((RegH*)h)->r.processUnorderedSweep(loam::Time(), xyz, n, loam::b200::RingLayout(lower_bound_deg, upper_bound_deg,
                                                                                      (uint16_t)n_rings));
    return 0;
  });
}
int loam_b200_scanreg_cloud_size(void* h, int which) { return (int)((RegH*)h)->cloud(which).size(); }
int loam_b200_scanreg_cloud_copy(void* h, int which, float* out) { dump(((RegH*)h)->cloud(which), out); return 0; }
int loam_b200_scanreg_index_size(void* h, int which) { return (int)((RegH*)h)->index(which).size(); }
int loam_b200_scanreg_index_copy(void* h, int which, int* out) {
  const auto& v = ((RegH*)h)->index(which);
  if (!v.empty()) std::memcpy(out, v.data(), v.size() * sizeof(int));
  return 0;
}

void* loam_b200_odom_create(float scanPeriod, int maxIterations) { return new OdomH(scanPeriod, maxIterations); }
void loam_b200_odom_destroy(void* h) { delete (OdomH*)h; }
int loam_b200_odom_set_inputs(void* h, const float* sharp, int n_sharp, const float* less_sharp, int n_less_sharp,
                              const float* flat, int n_flat, const float* less_flat, int n_less_flat,
                              const float* full, int n_full) {
  return guarded([&] {
    auto& o = ((OdomH*)h)->o;
    fill(*o.cornerPointsSharp(), sharp, n_sharp);
    fill(*o.cornerPointsLessSharp(), less_sharp, n_less_sharp);
    fill(*o.surfPointsFlat(), flat, n_flat);
    fill(*o.surfPointsLessFlat(), less_flat, n_less_flat);
    fill(*o.laserCloud(), full, n_full);
    return 0;
  });
}
int loam_b200_odom_process(void* h) { return guarded([&] { ((OdomH*)h)->o.process(); return 0; }); }
int loam_b200_odom_full_to_end(void* h) {
  return guarded([&] { auto& o = ((OdomH*)h)->o; o.transformToEnd(o.laserCloud()); return 0; });
}
int loam_b200_odom_get_twist(void* h, int which, float* out6) {
  auto& o = ((OdomH*)h)->o;
  twist6(which == 0 ? o.transform() : o.transformSum(), out6);
  return 0;
}
int loam_b200_odom_cloud_size(void* h, int which) { return (int)((OdomH*)h)->cloud(which).size(); }
int loam_b200_odom_cloud_copy(void* h, int which, float* out) { dump(((OdomH*)h)->cloud(which), out); return 0; }
int loam_b200_odom_last_iterations(void* h) { return (int)((OdomH*)h)->o.lastIterationCount(); }

void* loam_b200_map_create(float scanPeriod, int maxIterations) { return new MapH(scanPeriod, maxIterations); }
void loam_b200_map_destroy(void* h) { delete (MapH*)h; }
int loam_b200_map_seed(void* h, const float* corner, int n_corner, const float* surf, int n_surf) {
  return guarded([&] {
    Cloud c, s;
    fill(c, corner, n_corner);
    fill(s, surf, n_surf);
    ((MapH*)h)->m.seedMap(c, s);
    return 0;
  });
}
int loam_b200_map_set_inputs(void* h, const float* corner_last, int n_corner, const float* surf_last, int n_surf,
                             const float* full, int n_full) {
  return guarded([&] {
    auto& m = ((MapH*)h)->m;
    fill(m.laserCloudCornerLast(), corner_last, n_corner);
    fill(m.laserCloudSurfLast(), surf_last, n_surf);
    fill(m.laserCloud(), full, n_full);
    return 0;
  });
}
int loam_b200_map_update_odometry(void* h, const float* s) {
  loam::Twist t;
  t.rot_x = s[0]; t.rot_y = s[1]; t.rot_z = s[2];
  t.pos = loam::Vector3(s[3], s[4], s[5]);
  ((MapH*)h)->m.updateOdometry(t);
  return 0;
}
int loam_b200_map_process(void* h) {
  return guarded([&] { return ((MapH*)h)->m.process(loam::Time()) ? 1 : 0; });
}
int loam_b200_map_get_twist(void* h, int which, float* out6) {
  auto& m = ((MapH*)h)->m;
  twist6(which == 0 ? m.transformAftMapped() : which == 1 ? m.transformBefMapped() : m.transformTobeMapped(), out6);
  return 0;
}
int loam_b200_map_cloud_size(void* h, int which) { return (int)((MapH*)h)->cloud(which).size(); }
int loam_b200_map_cloud_copy(void* h, int which, float* out) { dump(((MapH*)h)->cloud(which), out); return 0; }
int loam_b200_map_last_iterations(void* h) { return (int)((MapH*)h)->m.lastIterationCount(); }
int loam_b200_map_retain_from_map(void* h, int on) {
  return guarded([&] { ((MapH*)h)->m.retainFromMapClouds(on != 0); return 0; });
}
int loam_b200_map_dense_enable(void* h, float leaf, long long max_voxels) {
  if (const int rc = map_in_flight((MapH*)h)) return rc;
  return guarded([&] { ((MapH*)h)->m.enableDenseMap(leaf, max_voxels); return 0; });
}
int loam_b200_map_dense_stats(void* h, long long* out3) {
  if (const int rc = map_in_flight((MapH*)h)) return rc;
  return guarded([&] {
    const auto s = ((MapH*)h)->m.denseMapStats();
    out3[0] = s.voxels; out3[1] = s.skipped; out3[2] = s.dropped;
    return 0;
  });
}
int loam_b200_map_dense_export(void* h, float* xyzi, unsigned int* counts, int cap, int* n_out) {
  if (const int rc = map_in_flight((MapH*)h)) return rc;
  return guarded([&] {
    auto* m = (MapH*)h;
    std::vector<uint32_t> cnt;
    m->m.denseMap(m->scratchA, counts ? &cnt : nullptr);
    const int n = (int)m->scratchA.points.size();
    *n_out = n;
    if (n > cap) { g_err = "loam_b200_map_dense_export: output capacity too small"; return (int)LOAM_B200_ERR_CAPACITY; }
    dump(m->scratchA, xyzi);
    if (counts && n > 0) std::memcpy(counts, cnt.data(), (size_t)n * sizeof(uint32_t));
    return 0;
  });
}
int loam_b200_map_dense_visibility(void* h, double h_res_deg, double v_res_deg, double margin) {
  if (const int rc = map_in_flight((MapH*)h)) return rc;
  return guarded([&] { ((MapH*)h)->m.enableDenseVisibility(h_res_deg, v_res_deg, margin); return 0; });
}
int loam_b200_map_dense_carving(void* h, double margin, double max_range) {
  if (const int rc = map_in_flight((MapH*)h)) return rc;
  return guarded([&] { ((MapH*)h)->m.enableDenseCarving(margin, max_range); return 0; });
}
int loam_b200_map_dense_export_filtered(void* h, double max_miss_ratio, float* xyzi, unsigned int* counts,
                                        unsigned short* hits, unsigned short* misses, int cap, int* n_out) {
  if (const int rc = map_in_flight((MapH*)h)) return rc;
  return guarded([&] {
    auto* m = (MapH*)h;
    std::vector<uint32_t> cnt;
    std::vector<uint16_t> hit, miss;
    m->m.denseMapFiltered(m->scratchA, max_miss_ratio, counts ? &cnt : nullptr, hits ? &hit : nullptr, misses ? &miss : nullptr);
    const int n = (int)m->scratchA.points.size();
    *n_out = n;
    if (n > cap) {
      g_err = "loam_b200_map_dense_export_filtered: output capacity too small";
      return (int)LOAM_B200_ERR_CAPACITY;
    }
    dump(m->scratchA, xyzi);
    if (counts && n > 0) std::memcpy(counts, cnt.data(), (size_t)n * sizeof(uint32_t));
    if (hits && n > 0) std::memcpy(hits, hit.data(), (size_t)n * sizeof(uint16_t));
    if (misses && n > 0) std::memcpy(misses, miss.data(), (size_t)n * sizeof(uint16_t));
    return 0;
  });
}
int loam_b200_map_dense_export_normals(void* h, double max_miss_ratio, int radius, const double* viewpoint,
                                       float* xyzi, unsigned int* counts, float* normals, int cap, int* n_out) {
  if (const int rc = map_in_flight((MapH*)h)) return rc;
  if (!viewpoint) { g_err = "loam_b200_map_dense_export_normals: viewpoint is NULL"; return (int)LOAM_B200_ERR_ARG; }
  return guarded([&] {
    auto* m = (MapH*)h;
    std::vector<uint32_t> cnt;
    pcl::PointCloud<pcl::PointXYZINormal> cloud;
    m->m.denseMapNormals(cloud, max_miss_ratio, radius, viewpoint, counts ? &cnt : nullptr);
    const int n = (int)cloud.points.size();
    *n_out = n;
    if (n > cap) {
      g_err = "loam_b200_map_dense_export_normals: output capacity too small";
      return (int)LOAM_B200_ERR_CAPACITY;
    }
    for (int i = 0; i < n; i++) {
      const pcl::PointXYZINormal& p = cloud.points[(size_t)i];
      const float a[4] = {p.x, p.y, p.z, p.intensity}, b[4] = {p.normal_x, p.normal_y, p.normal_z, p.curvature};
      std::memcpy(xyzi + 4 * i, a, sizeof(a));
      std::memcpy(normals + 4 * i, b, sizeof(b));
    }
    if (counts && n > 0) std::memcpy(counts, cnt.data(), (size_t)n * sizeof(uint32_t));
    return 0;
  });
}
int loam_b200_map_dense_snapshot(void* h, unsigned long long* keys, unsigned int* counts, unsigned short* hits,
                                 unsigned short* misses, double* sums, int cap, int* n_out) {
  if (const int rc = map_in_flight((MapH*)h)) return rc;
  if (!n_out || cap < 0) { g_err = "loam_b200_map_dense_snapshot: bad capacity or NULL n_out"; return (int)LOAM_B200_ERR_ARG; }
  return guarded([&] {
    loam::BasicLaserMapping::DenseMapSnapshot s;
    ((MapH*)h)->m.denseMapSnapshot(s);
    const int n = (int)s.counts.size();
    *n_out = n;
    if (n > cap) { g_err = "loam_b200_map_dense_snapshot: output capacity too small"; return (int)LOAM_B200_ERR_CAPACITY; }
    if (n == 0) return 0;
    if (!counts || !sums) { g_err = "loam_b200_map_dense_snapshot: counts or sums is NULL"; return (int)LOAM_B200_ERR_ARG; }
    if (keys) std::memcpy(keys, s.keys.data(), (size_t)n * sizeof(uint64_t));
    std::memcpy(counts, s.counts.data(), (size_t)n * sizeof(uint32_t));
    if (hits) std::memcpy(hits, s.hits.data(), (size_t)n * sizeof(uint16_t));
    if (misses) std::memcpy(misses, s.misses.data(), (size_t)n * sizeof(uint16_t));
    std::memcpy(sums, s.sums.data(), (size_t)n * 4 * sizeof(double));
    return 0;
  });
}
static std::vector<loam::Twist> twists_of(const float* t6, int k);
int loam_b200_map_dense_merge(void* h, const unsigned int* counts, const unsigned short* hits,
                              const unsigned short* misses, const double* sums, int n, const float* pose6) {
  if (const int rc = map_in_flight((MapH*)h)) return rc;
  if (n < 0 || (n > 0 && (!counts || !hits || !misses || !sums))) {
    g_err = "loam_b200_map_dense_merge: bad size or NULL argument";
    return (int)LOAM_B200_ERR_ARG;
  }
  return guarded([&] {
    loam::BasicLaserMapping::DenseMapSnapshot s;
    s.counts.assign(counts, counts + n);
    s.hits.assign(hits, hits + n);
    s.misses.assign(misses, misses + n);
    s.sums.assign(sums, sums + 4 * (size_t)n);
    if (pose6) {
      const loam::Twist t = twists_of(pose6, 1)[0];
      ((MapH*)h)->m.mergeDenseMap(s, &t);
    } else {
      ((MapH*)h)->m.mergeDenseMap(s, nullptr);
    }
    return 0;
  });
}
int loam_b200_map_dense_target_build(void* h, double max_miss_ratio, int radius, const double* viewpoint, int* n_out) {
  if (const int rc = map_in_flight((MapH*)h)) return rc;
  if (!viewpoint || !n_out) { g_err = "loam_b200_map_dense_target_build: NULL argument"; return (int)LOAM_B200_ERR_ARG; }
  return guarded([&] {
    *n_out = (int)((MapH*)h)->m.buildDenseTarget(max_miss_ratio, radius, viewpoint);
    return 0;
  });
}
int loam_b200_map_dense_target_load(void* h, float leaf, const float* xyzi, const float* normals, int n) {
  if (const int rc = map_in_flight((MapH*)h)) return rc;
  if (n < 0 || (n > 0 && (!xyzi || !normals))) {
    g_err = "loam_b200_map_dense_target_load: bad size or NULL argument";
    return (int)LOAM_B200_ERR_ARG;
  }
  return guarded([&] {
    pcl::PointCloud<pcl::PointXYZINormal> target;
    target.points.resize((size_t)n);
    for (int i = 0; i < n; i++) {
      pcl::PointXYZINormal& p = target.points[(size_t)i];
      p.x = xyzi[4 * i + 0]; p.y = xyzi[4 * i + 1]; p.z = xyzi[4 * i + 2]; p.intensity = xyzi[4 * i + 3];
      p.normal_x = normals[4 * i + 0]; p.normal_y = normals[4 * i + 1]; p.normal_z = normals[4 * i + 2];
      p.curvature = normals[4 * i + 3];
    }
    ((MapH*)h)->m.loadDenseTarget(leaf, target);
    return 0;
  });
}
int loam_b200_map_dense_align(void* h, const float* xyzi, int n, const float* initial6, int search_radius,
                              int max_iterations, float* twist_out6, int* stats_out4, float* rms_out) {
  if (const int rc = map_in_flight((MapH*)h)) return rc;
  if (n < 0 || (n > 0 && !xyzi) || !initial6 || !twist_out6) {
    g_err = "loam_b200_map_dense_align: bad size or NULL argument";
    return (int)LOAM_B200_ERR_ARG;
  }
  return guarded([&] {
    auto* m = (MapH*)h;
    fill(m->scratchA, xyzi, n);
    loam::Twist initial;
    initial.rot_x = initial6[0];
    initial.rot_y = initial6[1];
    initial.rot_z = initial6[2];
    initial.pos.x() = initial6[3];
    initial.pos.y() = initial6[4];
    initial.pos.z() = initial6[5];
    const auto r = m->m.alignToDenseTarget(m->scratchA, initial, search_radius, max_iterations);
    twist6(r.pose, twist_out6);
    if (stats_out4) {
      stats_out4[0] = (int)r.iterations;
      stats_out4[1] = (int)r.nSelected;
      stats_out4[2] = r.degenerate ? 1 : 0;
      stats_out4[3] = r.converged ? 1 : 0;
    }
    if (rms_out) *rms_out = r.rms;
    return 0;
  });
}
static std::vector<loam::Twist> twists_of(const float* t6, int k) {
  std::vector<loam::Twist> out((size_t)k);
  for (int h = 0; h < k; h++) {
    const float* t = t6 + 6 * h;
    out[(size_t)h].rot_x = t[0];
    out[(size_t)h].rot_y = t[1];
    out[(size_t)h].rot_z = t[2];
    out[(size_t)h].pos = loam::Vector3(t[3], t[4], t[5]);
  }
  return out;
}
static void align_result_of(const loam::BasicLaserMapping::DenseAlignResult& r, loam_b200_align_result& o) {
  o.rot[0] = r.pose.rot_x.rad(); o.rot[1] = r.pose.rot_y.rad(); o.rot[2] = r.pose.rot_z.rad();
  o.pos[0] = r.pose.pos.x(); o.pos[1] = r.pose.pos.y(); o.pos[2] = r.pose.pos.z();
  o.iterations = (int)r.iterations;
  o.n_selected = (int)r.nSelected;
  o.rms = r.rms;
  o.degenerate = r.degenerate ? 1 : 0;
  o.converged = r.converged ? 1 : 0;
}
int loam_b200_map_dense_score(void* h, const float* xyzi, int n, const float* poses6, int k, int search_radius,
                              int* n_selected, float* sum_pd2_sq) {
  if (const int rc = map_in_flight((MapH*)h)) return rc;
  if (n < 0 || (n > 0 && !xyzi) || !poses6 || k < 1 || !n_selected || !sum_pd2_sq) {
    g_err = "loam_b200_map_dense_score: bad size or NULL argument";
    return (int)LOAM_B200_ERR_ARG;
  }
  return guarded([&] {
    auto* m = (MapH*)h;
    fill(m->scratchA, xyzi, n);
    const auto r = m->m.scoreDenseTarget(m->scratchA, twists_of(poses6, k), search_radius);
    for (int i = 0; i < k; i++) {
      n_selected[i] = (int)r[(size_t)i].nSelected;
      sum_pd2_sq[i] = r[(size_t)i].sumPd2Sq;
    }
    return 0;
  });
}
int loam_b200_map_dense_align_batch(void* h, const float* xyzi, int n, const float* initial6, int k, int search_radius,
                                    int max_iterations, float* twist_out6, int* stats_out4, float* rms_out) {
  if (const int rc = map_in_flight((MapH*)h)) return rc;
  if (n < 0 || (n > 0 && !xyzi) || !initial6 || k < 1 || !twist_out6) {
    g_err = "loam_b200_map_dense_align_batch: bad size or NULL argument";
    return (int)LOAM_B200_ERR_ARG;
  }
  return guarded([&] {
    auto* m = (MapH*)h;
    fill(m->scratchA, xyzi, n);
    const auto r = m->m.alignToDenseTarget(m->scratchA, twists_of(initial6, k), search_radius, max_iterations);
    for (int i = 0; i < k; i++) {
      twist6(r[(size_t)i].pose, twist_out6 + 6 * i);
      if (stats_out4) {
        stats_out4[4 * i + 0] = (int)r[(size_t)i].iterations;
        stats_out4[4 * i + 1] = (int)r[(size_t)i].nSelected;
        stats_out4[4 * i + 2] = r[(size_t)i].degenerate ? 1 : 0;
        stats_out4[4 * i + 3] = r[(size_t)i].converged ? 1 : 0;
      }
      if (rms_out) rms_out[i] = r[(size_t)i].rms;
    }
    return 0;
  });
}
int loam_b200_map_dense_relocalize(void* h, const float* xyzi, int n, const float* hyps6, int k,
                                   const loam_b200_reloc_params* prm, loam_b200_reloc_candidate* out, int cap,
                                   int* n_out) {
  if (const int rc = map_in_flight((MapH*)h)) return rc;
  if (n < 0 || (n > 0 && !xyzi) || !hyps6 || k < 1 || !prm || !out || cap < 1 || !n_out) {
    g_err = "loam_b200_map_dense_relocalize: bad size or NULL argument";
    return (int)LOAM_B200_ERR_ARG;
  }
  return guarded([&] {
    auto* m = (MapH*)h;
    fill(m->scratchA, xyzi, n);
    loam::BasicLaserMapping::RelocParams p;
    p.scoreRadius = prm->score_radius;
    p.coarseRadius = prm->coarse_radius;
    p.fineRadius = prm->fine_radius;
    p.keep = prm->keep;
    p.maxIterations = prm->max_iterations;
    p.dedupMetres = prm->dedup_m;
    p.dedupDegrees = prm->dedup_deg;
    const auto r = m->m.relocalizeInDenseTarget(m->scratchA, twists_of(hyps6, k), p, (size_t)cap);
    *n_out = (int)r.size();
    for (size_t i = 0; i < r.size(); i++) {
      out[i].hypothesis = (int)r[i].hypothesis;
      out[i].score_selected = (int)r[i].scoreSelected;
      align_result_of(r[i].coarse, out[i].coarse);
      align_result_of(r[i].fine, out[i].fine);
      out[i].selected = (int)r[i].selected;
      out[i].rms = r[i].rms;
    }
    return 0;
  });
}
int loam_b200_map_dense_raycast(void* h, const float* rays, int n, const float* pose6, float min_range,
                                float max_range, float* range, int* index) {
  if (const int rc = map_in_flight((MapH*)h)) return rc;
  if (n < 0 || (n > 0 && (!rays || !range)) || !pose6) {
    g_err = "loam_b200_map_dense_raycast: bad size or NULL argument";
    return (int)LOAM_B200_ERR_ARG;
  }
  return guarded([&] {
    auto* m = (MapH*)h;
    fill(m->scratchA, rays, n);
    std::vector<float> r;
    std::vector<int> idx;
    m->m.raycastDenseTarget(m->scratchA, twists_of(pose6, 1)[0], min_range, max_range, r, index ? &idx : nullptr);
    if (n > 0) std::memcpy(range, r.data(), (size_t)n * sizeof(float));
    if (index && n > 0) std::memcpy(index, idx.data(), (size_t)n * sizeof(int));
    return 0;
  });
}
int loam_b200_map_dense_distance_build(void* h, const int* lo, const int* dims, float max_distance, float* dist,
                                       int* sq) {
  if (const int rc = map_in_flight((MapH*)h)) return rc;
  if (!lo || !dims) {
    g_err = "loam_b200_map_dense_distance_build: NULL argument";
    return (int)LOAM_B200_ERR_ARG;
  }
  return guarded([&] {
    auto* m = (MapH*)h;
    std::vector<float> d;
    std::vector<int> s;
    m->m.buildDenseDistanceField(lo, dims, max_distance, dist ? &d : nullptr, sq ? &s : nullptr);
    if (dist) std::memcpy(dist, d.data(), d.size() * sizeof(float));
    if (sq) std::memcpy(sq, s.data(), s.size() * sizeof(int));
    return 0;
  });
}
int loam_b200_map_dense_distance_query(void* h, const float* xyzi, int n, float* dist, float* grad) {
  if (const int rc = map_in_flight((MapH*)h)) return rc;
  if (n < 0 || (n > 0 && (!xyzi || !dist))) {
    g_err = "loam_b200_map_dense_distance_query: bad size or NULL argument";
    return (int)LOAM_B200_ERR_ARG;
  }
  return guarded([&] {
    auto* m = (MapH*)h;
    fill(m->scratchA, xyzi, n);
    std::vector<float> d, g;
    m->m.queryDenseDistance(m->scratchA, d, grad ? &g : nullptr);
    if (n > 0) std::memcpy(dist, d.data(), (size_t)n * sizeof(float));
    if (grad && n > 0) std::memcpy(grad, g.data(), (size_t)3 * n * sizeof(float));
    return 0;
  });
}
int loam_b200_map_dense_target_size(void* h, int* n_out) {
  if (const int rc = map_in_flight((MapH*)h)) return rc;
  if (!n_out) {
    g_err = "loam_b200_map_dense_target_size: NULL argument";
    return (int)LOAM_B200_ERR_ARG;
  }
  return guarded([&] {
    *n_out = (int)((MapH*)h)->m.denseTargetSize();
    return 0;
  });
}
// the records and labels of a target segmentation by the drop-in class: ERR_CAPACITY when they exceed cap
static int put_segments(const char* what, const std::vector<loam::BasicLaserMapping::DenseSegment>& seg,
                        const std::vector<int>& lab, int* labels, loam_b200_segment* segments, int cap, int* n_out) {
  *n_out = (int)seg.size();
  if ((int)seg.size() > cap) {
    g_err = std::string(what) + ": output capacity too small";
    return (int)LOAM_B200_ERR_CAPACITY;
  }
  for (size_t i = 0; i < seg.size(); i++) {
    segments[i].size = (int32_t)seg[i].size;
    segments[i].first = (int32_t)seg[i].first;
    for (int a = 0; a < 3; a++) {
      segments[i].lo[a] = seg[i].lo[a];
      segments[i].hi[a] = seg[i].hi[a];
      segments[i].centroid[a] = seg[i].centroid[a];
    }
  }
  if (labels && !lab.empty()) std::memcpy(labels, lab.data(), lab.size() * sizeof(int));
  return 0;
}
int loam_b200_map_dense_segment(void* h, float tol, int min_size, int max_size, int* labels,
                                loam_b200_segment* segments, int cap, int* n_out) {
  if (const int rc = map_in_flight((MapH*)h)) return rc;
  if (cap < 0 || (cap > 0 && !segments) || !n_out) {
    g_err = "loam_b200_map_dense_segment: bad size or NULL argument";
    return (int)LOAM_B200_ERR_ARG;
  }
  return guarded([&] {
    auto* m = (MapH*)h;
    std::vector<int> lab;
    const auto seg = m->m.segmentDenseTarget(tol, min_size, max_size, labels ? &lab : nullptr);
    return put_segments("loam_b200_map_dense_segment", seg, lab, labels, segments, cap, n_out);
  });
}
int loam_b200_map_dense_ground(void* h, const loam_b200_ground_params* params, int* labels,
                               loam_b200_segment* patches, int cap, int* n_out) {
  if (const int rc = map_in_flight((MapH*)h)) return rc;
  if (!params || cap < 0 || (cap > 0 && !patches) || !n_out) {
    g_err = "loam_b200_map_dense_ground: bad size or NULL argument";
    return (int)LOAM_B200_ERR_ARG;
  }
  return guarded([&] {
    auto* m = (MapH*)h;
    loam::BasicLaserMapping::DenseGroundParams prm;
    prm.maxSlopeDeg = params->max_slope_deg;
    prm.maxCurvature = params->max_curvature;
    prm.tolerance = params->tol;
    prm.maxStep = params->max_step;
    prm.minSize = params->min_size;
    std::vector<int> lab;
    const auto seg = m->m.groundDenseTarget(prm, labels ? &lab : nullptr);
    return put_segments("loam_b200_map_dense_ground", seg, lab, labels, patches, cap, n_out);
  });
}
int loam_b200_map_dense_segment_above_ground(void* h, float tol, int min_size, int max_size, int* labels,
                                             loam_b200_segment* segments, int cap, int* n_out) {
  if (const int rc = map_in_flight((MapH*)h)) return rc;
  if (cap < 0 || (cap > 0 && !segments) || !n_out) {
    g_err = "loam_b200_map_dense_segment_above_ground: bad size or NULL argument";
    return (int)LOAM_B200_ERR_ARG;
  }
  return guarded([&] {
    auto* m = (MapH*)h;
    std::vector<int> lab;
    const auto seg = m->m.segmentDenseTargetAboveGround(tol, min_size, max_size, labels ? &lab : nullptr);
    return put_segments("loam_b200_map_dense_segment_above_ground", seg, lab, labels, segments, cap, n_out);
  });
}
int loam_b200_map_dense_ground_cloud(void* h, const float* xyzi, int n, const float* pose6, int search_radius,
                                     float max_height, float* ground, int* n_ground, float* nonground,
                                     int* n_nonground) {
  if (const int rc = map_in_flight((MapH*)h)) return rc;
  if (n < 0 || (n > 0 && !xyzi) || !pose6 || !n_ground || !n_nonground) {
    g_err = "loam_b200_map_dense_ground_cloud: bad size or NULL argument";
    return (int)LOAM_B200_ERR_ARG;
  }
  return guarded([&] {
    auto* m = (MapH*)h;
    fill(m->scratchA, xyzi, n);
    Cloud g, ng;
    m->m.splitGround(m->scratchA, twists_of(pose6, 1)[0], g, ng, search_radius, max_height);
    *n_ground = (int)g.points.size();
    *n_nonground = (int)ng.points.size();
    if (ground) dump(g, ground);
    if (nonground) dump(ng, nonground);
    return 0;
  });
}
static loam::BasicLaserMapping::PlaceParams place_params_of(const loam_b200_place_params& p) {
  loam::BasicLaserMapping::PlaceParams o;
  o.rings = p.rings;
  o.sectors = p.sectors;
  o.maxRadius = p.max_radius;
  o.heightOffset = p.height_offset;
  o.minRange = p.min_range;
  o.maxRange = p.max_range;
  return o;
}
static void place_match_of(const loam::BasicLaserMapping::PlaceMatch& m, loam_b200_place_match& o) {
  o.candidate = (int)m.candidate;
  o.shift = m.shift;
  o.yaw = m.yaw;
  o.pos[0] = m.position.x(); o.pos[1] = m.position.y(); o.pos[2] = m.position.z();
  o.dist = m.dist;
}
int loam_b200_map_dense_place_build(void* h, const float* positions, int k, const float* rays, int n_rays,
                                    const loam_b200_place_params* prm) {
  if (const int rc = map_in_flight((MapH*)h)) return rc;
  if (k < 1 || !positions || n_rays < 0 || (n_rays > 0 && !rays) || !prm) {
    g_err = "loam_b200_map_dense_place_build: bad size or NULL argument";
    return (int)LOAM_B200_ERR_ARG;
  }
  return guarded([&] {
    auto* m = (MapH*)h;
    fill(m->scratchA, rays, n_rays);
    std::vector<loam::Vector3> pos((size_t)k);
    for (int i = 0; i < k; i++) pos[(size_t)i] = loam::Vector3(positions[3 * i], positions[3 * i + 1], positions[3 * i + 2]);
    m->m.buildDensePlaces(pos, m->scratchA, place_params_of(*prm));
    return 0;
  });
}
int loam_b200_map_dense_place_query(void* h, const float* xyzi, int n, int top_m, loam_b200_place_match* out,
                                    int* n_out) {
  if (const int rc = map_in_flight((MapH*)h)) return rc;
  if (n < 0 || (n > 0 && !xyzi) || top_m < 1 || !out || !n_out) {
    g_err = "loam_b200_map_dense_place_query: bad size or NULL argument";
    return (int)LOAM_B200_ERR_ARG;
  }
  return guarded([&] {
    auto* m = (MapH*)h;
    fill(m->scratchA, xyzi, n);
    const auto r = m->m.queryDensePlaces(m->scratchA, (size_t)top_m);
    *n_out = (int)r.size();
    for (size_t i = 0; i < r.size(); i++) place_match_of(r[i], out[i]);
    return 0;
  });
}
int loam_b200_map_dense_relocalize_global(void* h, const float* xyzi, int n, int top_m, float yaw_step_deg,
                                          int yaw_steps, float xz_step, int xz_steps,
                                          const loam_b200_reloc_params* prm, loam_b200_reloc_candidate* out, int cap,
                                          int* n_out) {
  if (const int rc = map_in_flight((MapH*)h)) return rc;
  if (n < 0 || (n > 0 && !xyzi) || top_m < 1 || !prm || !out || cap < 1 || !n_out) {
    g_err = "loam_b200_map_dense_relocalize_global: bad size or NULL argument";
    return (int)LOAM_B200_ERR_ARG;
  }
  return guarded([&] {
    auto* m = (MapH*)h;
    fill(m->scratchA, xyzi, n);
    loam::BasicLaserMapping::RelocParams p;
    p.scoreRadius = prm->score_radius;
    p.coarseRadius = prm->coarse_radius;
    p.fineRadius = prm->fine_radius;
    p.keep = prm->keep;
    p.maxIterations = prm->max_iterations;
    p.dedupMetres = prm->dedup_m;
    p.dedupDegrees = prm->dedup_deg;
    loam::BasicLaserMapping::GlobalGrid g;
    g.topM = top_m;
    g.yawStepDeg = yaw_step_deg;
    g.yawSteps = yaw_steps;
    g.xzStep = xz_step;
    g.xzSteps = xz_steps;
    const auto r = m->m.relocalizeGlobalInDenseTarget(m->scratchA, g, p, (size_t)cap);
    *n_out = (int)r.size();
    for (size_t i = 0; i < r.size(); i++) {
      out[i].hypothesis = (int)r[i].hypothesis;
      out[i].score_selected = (int)r[i].scoreSelected;
      align_result_of(r[i].coarse, out[i].coarse);
      align_result_of(r[i].fine, out[i].fine);
      out[i].selected = (int)r[i].selected;
      out[i].rms = r[i].rms;
    }
    return 0;
  });
}
int loam_b200_map_debug_dense_table_slots(void* h, long long* out) {
  if (const int rc = map_in_flight((MapH*)h)) return rc;
  return guarded([&] { *out = ((MapH*)h)->m.denseTableSlots(); return 0; });
}
int loam_b200_map_dense_clear(void* h) {
  if (const int rc = map_in_flight((MapH*)h)) return rc;
  return guarded([&] { ((MapH*)h)->m.clearDenseMap(); return 0; });
}
int loam_b200_map_last_phase_seconds(void* h, double* out4) {
  const double* p = ((MapH*)h)->m.lastPhaseSeconds();
  for (int i = 0; i < 4; i++) out4[i] = p[i];
  return 0;
}

void* loam_b200_pipeline_create(float scanPeriod, int odomMaxIter, int mapMaxIter) {
  return new PipeH(scanPeriod, odomMaxIter, mapMaxIter);
}
void loam_b200_pipeline_destroy(void* h) { delete (PipeH*)h; }
int loam_b200_pipeline_seed_map(void* h, const float* corner, int n_corner, const float* surf, int n_surf) {
  return loam_b200_map_seed(&((PipeH*)h)->map, corner, n_corner, surf, n_surf);
}
int loam_b200_host_nccl_unique_id(unsigned char* out128) {
  const int rc = loam_b200_comm_unique_id(out128);
  if (rc) g_err = std::string("loam_b200_comm_unique_id: ") + loam_b200_strerror(rc);
  return rc;
}
int loam_b200_map_enable_sharding(void* h, int rank, int world, const unsigned char* nccl_id128) {
  return guarded([&] { ((MapH*)h)->m.enableSharding(rank, world, nccl_id128); return 0; });
}
// The scan-to-map iteration kernel exactly as this object launches it (its own context, persistent map store, the queries
// of the last process() call), timed with CUDA events over `reps` launches at the current mapped pose.
// out5: average launch microseconds, queries, table probes per query, candidate points per query, selected correspondences
int loam_b200_map_kernel_profile(void* h, int reps, double* out5) {
  return guarded([&] {
    auto& m = ((MapH*)h)->m;
    loam_b200_ctx* c = m.deviceContext()->get();
    auto ck = [&](int rc, const char* what) { m.deviceContext()->check(rc, what); };
    loam_b200_pose pose;
    b200::fillPose(m.transformAftMapped(), pose);
    loam_b200_normal_eq ne;
    unsigned long long probes = 0, cands = 0;
    ck(loam_b200_map_iterate_stats(c, &pose, &ne, &probes, &cands), "loam_b200_map_iterate_stats");
    for (int i = 0; i < 5; i++) ck(loam_b200_map_iterate(c, &pose, &ne), "loam_b200_map_iterate");
    ck(loam_b200_profile_reset(c), "loam_b200_profile_reset");
    ck(loam_b200_profile_enable(c, 1), "loam_b200_profile_enable");
    for (int i = 0; i < reps; i++) ck(loam_b200_map_iterate(c, &pose, &ne), "loam_b200_map_iterate");
    double ms = 0.0;
    long long launches = 0;
    ck(loam_b200_profile_get(c, LOAM_B200_K_MAP_ITER, &ms, &launches), "loam_b200_profile_get");
    ck(loam_b200_profile_enable(c, 0), "loam_b200_profile_enable");
    const double nq = (double)(m.cornerStackSize() + m.surfStackSize());
    out5[0] = launches > 0 ? 1e3 * ms / (double)launches : 0.0;
    out5[1] = nq;
    out5[2] = nq > 0 ? (double)probes / nq : 0.0;
    out5[3] = nq > 0 ? (double)cands / nq : 0.0;
    out5[4] = (double)ne.n_selected;
    return 0;
  });
}

// The same kernel on caller-supplied queries (map frame, identity pose) against this object's persistent map: the
// bandwidth stress of BASELINE config 5 -- queries spread over a map far larger than L2.  out5 as above.
int loam_b200_map_kernel_profile_queries(void* h, const float* queries, int n, int reps, double* out5) {
  return guarded([&] {
    auto& m = ((MapH*)h)->m;
    loam_b200_ctx* c = m.deviceContext()->get();
    auto ck = [&](int rc, const char* what) { m.deviceContext()->check(rc, what); };
    ck(loam_b200_map_set_queries(c, nullptr, 0, queries, n), "loam_b200_map_set_queries");
    loam::Twist identity;
    loam_b200_pose pose;
    b200::fillPose(identity, pose);
    loam_b200_normal_eq ne;
    unsigned long long probes = 0, cands = 0;
    ck(loam_b200_map_iterate_stats(c, &pose, &ne, &probes, &cands), "loam_b200_map_iterate_stats");
    for (int i = 0; i < 3; i++) ck(loam_b200_map_iterate(c, &pose, &ne), "loam_b200_map_iterate");
    ck(loam_b200_profile_reset(c), "loam_b200_profile_reset");
    ck(loam_b200_profile_enable(c, 1), "loam_b200_profile_enable");
    for (int i = 0; i < reps; i++) ck(loam_b200_map_iterate(c, &pose, &ne), "loam_b200_map_iterate");
    double ms = 0.0;
    long long launches = 0;
    ck(loam_b200_profile_get(c, LOAM_B200_K_MAP_ITER, &ms, &launches), "loam_b200_profile_get");
    ck(loam_b200_profile_enable(c, 0), "loam_b200_profile_enable");
    out5[0] = launches > 0 ? 1e3 * ms / (double)launches : 0.0;
    out5[1] = (double)n;
    out5[2] = n > 0 ? (double)probes / n : 0.0;
    out5[3] = n > 0 ? (double)cands / n : 0.0;
    out5[4] = (double)ne.n_selected;
    return 0;
  });
}

int loam_b200_map_peer_export(void* h, unsigned char* out64) {
  return guarded([&] { ((MapH*)h)->m.exportPeerHandle(out64); return 0; });
}
int loam_b200_map_enable_cube_sharding(void* h, int rank, int world, const unsigned char* handles, int slab_metres) {
  return guarded([&] { ((MapH*)h)->m.enableCubeSharding(rank, world, handles, slab_metres); return 0; });
}
// unmap the peers' inboxes (call on every rank, then synchronise the ranks, BEFORE any rank destroys its object: memory
// exported over CUDA IPC must not be freed while another process still has it mapped)
int loam_b200_map_disable_cube_sharding(void* h) {
  return guarded([&] {
    auto* ctx = ((MapH*)h)->m.deviceContext();
    if (ctx->created()) ctx->check(loam_b200_peer_disconnect(ctx->get()), "loam_b200_peer_disconnect");
    return 0;
  });
}
int loam_b200_map_enable_cube_sharding_local(void** hs, int world, int slab_metres) {
  return guarded([&] {
    std::vector<loam::BasicLaserMapping*> objs((size_t)world);
    for (int r = 0; r < world; r++) objs[r] = &((MapH*)hs[r])->m;
    loam::BasicLaserMapping::enableCubeShardingLocal(objs.data(), world, slab_metres);
    return 0;
  });
}
void* loam_b200_pipeline_scanreg(void* h) { return &((PipeH*)h)->reg; }
void* loam_b200_pipeline_odom(void* h) { return &((PipeH*)h)->odom; }
void* loam_b200_pipeline_map(void* h) { return &((PipeH*)h)->map; }

static int pipeline_sweep_impl(PipeH* h, const float* pts, const void* d_pts, const int* ring_sizes, int n_rings,
                               float* odom_sum6, float* map_aft6, double* st) {
  const double t0 = now();
  if (d_pts)
    h->reg.r.processDeviceSweep(loam::Time(), d_pts, ring_sizes, n_rings);
  else
    h->reg.r.processPackedSweep(loam::Time(), pts, ring_sizes, n_rings);
  const double t1 = now();
  // ScanRegistration::publishResult -> LaserOdometry::*Handler upstream (five clouds + imuTrans over ROS topics):
  // here a device-to-device hand-off
  auto& o = h->odom.o;
  o.adopt(h->reg.r);
  const double t1b = now();
  o.process();
  const double t2 = now();
  o.transformLaserCloudToEnd();  // LaserOdometry::publishResult, LaserOdometry.cpp:326 upstream
  const double t3 = now();
  auto& m = h->map.m;
  m.adopt(o);                    // LaserOdometry::publishResult -> LaserMapping::*Handler upstream
  const double t3b = now();
  const int ok = m.process(loam::Time()) ? 1 : 0;
  const double t4 = now();
  static const bool trace = std::getenv("LOAM_B200_TRACE") != nullptr;
  if (trace) {
    const double* ph = m.lastPhaseSeconds();
    fprintf(stderr, "[pipe] reg %.0f | adopt %.0f odom %.0f | to-end %.0f | adopt %.0f map %.0f (begin %.0f lm %.0f end %.0f surround %.0f) us\n",
            (t1 - t0) * 1e6, (t1b - t1) * 1e6, (t2 - t1b) * 1e6, (t3 - t2) * 1e6, (t3b - t3) * 1e6, (t4 - t3b) * 1e6, ph[0] * 1e6,
            ph[1] * 1e6, ph[2] * 1e6, ph[3] * 1e6);
  }
  twist6(o.transformSum(), odom_sum6);
  twist6(m.transformAftMapped(), map_aft6);
  if (st) { st[0] = t1 - t0; st[1] = t2 - t1; st[2] = t3 - t2; st[3] = t4 - t3; st[4] = t4 - t0; }
  return ok;
}

int loam_b200_pipeline_sweep(void* hh, const float* pts, const int* ring_sizes, int n_rings, float* odom_sum6,
                             float* map_aft6, double* st) {
  return guarded([&] { return pipeline_sweep_impl((PipeH*)hh, pts, nullptr, ring_sizes, n_rings, odom_sum6, map_aft6, st); });
}

int loam_b200_pipeline_sweep_device(void* hh, const void* d_pts, const int* ring_sizes, int n_rings, float* odom_sum6,
                                    float* map_aft6, double* st) {
  return guarded([&] { return pipeline_sweep_impl((PipeH*)hh, nullptr, d_pts, ring_sizes, n_rings, odom_sum6, map_aft6, st); });
}

// the same chain through the reference's own entry points and host clouds only (what separate ROS nodes would do):
// processScanlines(vector<PointCloud>) -> host cloud copies -> process() -> host cloud copies -> process(Time)
int loam_b200_pipeline_sweep_hostclouds(void* hh, const float* pts, const int* ring_sizes, int n_rings, float* odom_sum6,
                                        float* map_aft6, double* st) {
  return guarded([&] {
    PipeH* h = (PipeH*)hh;
    const double t0 = now();
    h->reg.process(pts, ring_sizes, n_rings);
    const double t1 = now();
    auto& o = h->odom.o;
    *o.cornerPointsSharp() = h->reg.r.cornerPointsSharp();
    *o.cornerPointsLessSharp() = h->reg.r.cornerPointsLessSharp();
    *o.surfPointsFlat() = h->reg.r.surfacePointsFlat();
    *o.surfPointsLessFlat() = h->reg.r.surfacePointsLessFlat();
    *o.laserCloud() = h->reg.r.laserCloud();
    o.updateIMU(h->reg.r.imuTransform());
    o.process();
    const double t2 = now();
    o.transformToEnd(o.laserCloud());
    const double t3 = now();
    auto& m = h->map.m;
    m.laserCloudCornerLast() = *o.lastCornerCloud();
    m.laserCloudSurfLast() = *o.lastSurfaceCloud();
    m.laserCloud() = *o.laserCloud();
    m.updateOdometry(o.transformSum());
    const int ok = m.process(loam::Time()) ? 1 : 0;
    const double t4 = now();
    twist6(o.transformSum(), odom_sum6);
    twist6(m.transformAftMapped(), map_aft6);
    if (st) { st[0] = t1 - t0; st[1] = t2 - t1; st[2] = t3 - t2; st[3] = t4 - t3; st[4] = t4 - t0; }
    return ok;
  });
}

// everything enqueued or posted to helper threads by the three stage objects has finished on the GPU
int loam_b200_pipeline_sync(void* hh) {
  return guarded([&] {
    PipeH* h = (PipeH*)hh;
    b200::Context* cs[3] = {h->reg.r.deviceContext(), h->odom.o.deviceContext(), h->map.m.deviceContext()};
    for (auto* c : cs)
      if (c->created()) c->check(loam_b200_sync(c->get()), "loam_b200_sync");
    return 0;
  });
}

// ---- streaming form: the three stages work on consecutive sweeps concurrently (StreamRunner above) ----
int loam_b200_pipeline_submit(void* hh, const float* pts, const void* d_pts, const int* ring_sizes, int n_rings) {
  PipeH* h = (PipeH*)hh;
  if (!h || (!pts && !d_pts) || !ring_sizes || n_rings <= 0) { g_err = "invalid argument"; return -1; }
  if (!h->runner) {
    h->runner = new StreamRunner(h);
    h->map.runner = h->runner;
  }
  return h->runner->submit(pts, d_pts, ring_sizes, n_rings);
}

// out9: seconds the registration / odometry / mapping stage threads spent working, waiting for a neighbour stage, and in
// the adopt() hand-offs since the pipeline started streaming (call while no sweep is in flight); reset = clear afterwards
int loam_b200_pipeline_stage_seconds(void* hh, double* out9, int reset) {
  PipeH* h = (PipeH*)hh;
  if (!h || !out9) return -1;
  for (int i = 0; i < 9; i++) out9[i] = 0.0;
  if (!h->runner) return 0;
  std::lock_guard<std::mutex> lk(h->runner->m);
  for (int s = 0; s < 3; s++) {
    out9[s] = h->runner->busy[s];
    out9[3 + s] = h->runner->idle[s];
    out9[6 + s] = h->runner->handoff[s];
    if (reset) h->runner->busy[s] = h->runner->idle[s] = h->runner->handoff[s] = 0.0;
  }
  if (reset) h->runner->t_reset = now();
  return 0;
}

int loam_b200_pipeline_collect(void* hh, int wait, float* odom_sum6, float* map_aft6, int* ok) {
  PipeH* h = (PipeH*)hh;
  if (!h || !h->runner) return 0;
  SweepResult r;
  const int rc = h->runner->collect(wait, &r);
  if (rc == 1) {
    if (odom_sum6) std::memcpy(odom_sum6, r.odom, sizeof r.odom);
    if (map_aft6) std::memcpy(map_aft6, r.aft, sizeof r.aft);
    if (ok) *ok = r.ok;
  }
  return rc;
}

}  // extern "C"
