// Glue between the pcl::PointCloud-based Basic* classes and the C ABI (include/loam_b200.h).
// Nothing here computes on the CPU: a missing GPU / failed call surfaces as std::runtime_error from process*().
#pragma once
#include <cmath>
#include <cstdint>
#include <stdexcept>
#include <string>
#include <vector>

#include <pcl/point_cloud.h>
#include <pcl/filters/voxel_grid.h>

#include "loam_b200.h"
#include "loam_velodyne/Angle.h"
#include "loam_velodyne/Twist.h"

namespace loam {
namespace b200 {

// device selected for contexts created by the Basic* classes (default: $LOAM_B200_DEVICE, else $LOCAL_RANK, else 0)
int defaultDevice();
void setDefaultDevice(int device);

class Context {
 public:
  Context() : ctx_(nullptr), priority_(0) {}
  void setPriority(int level) { priority_ = level; }  // before first use (loam_b200_set_priority)
  ~Context() { if (ctx_) loam_b200_destroy(ctx_); }
  Context(const Context&) = delete;
  Context& operator=(const Context&) = delete;
  loam_b200_ctx* get();  // created on first use; throws when no GPU is usable
  bool created() const { return ctx_ != nullptr; }
  void check(int status, const char* what);

 private:
  loam_b200_ctx* ctx_;
  int priority_;
};

typedef pcl::PointCloud<pcl::PointXYZI> Cloud;

// A pcl cloud of the drop-in API whose authoritative copy may live in a cloud slot of a context (HBM).  The host
// pcl::PointCloud is only materialised when an accessor needs it; a mutable accessor marks the device copy stale so
// the next stage call re-uploads.  This is what lets registration -> odometry -> mapping chain without host hops
// while the reference's cloud accessors keep working.
class DualCloud {
 public:
  DualCloud() : host_(new Cloud()), ctx_(nullptr), slot_(-1), hostValid_(true), devValid_(false), devN_(0) {}
  void bind(Context* ctx, int slot) { ctx_ = ctx; slot_ = slot; }
  int slot() const { return slot_; }
  Context* context() const { return ctx_; }

  // the reference hands out `Ptr&` / `Cloud&`; callers may modify through them
  Cloud::Ptr& hostPtrMutable() { materialise(); devValid_ = false; return host_; }
  Cloud& hostMutable() { materialise(); devValid_ = false; return *host_; }
  const Cloud::Ptr& hostPtr() const { const_cast<DualCloud*>(this)->materialise(); return host_; }
  const Cloud& host() const { const_cast<DualCloud*>(this)->materialise(); return *host_; }

  std::size_t size() const { return hostValid_ ? host_->points.size() : (std::size_t)deviceCount(); }
  void deviceWritten(int n) { devValid_ = true; hostValid_ = false; devN_ = n; }
  // the device copy is being produced asynchronously: its size is asked from the context on first use
  void deviceWrittenLazy() { devValid_ = true; hostValid_ = false; devN_ = -1; }
  int deviceCount() const;
  void ensureDevice();   // upload when the device copy is stale
  void materialise();    // download when the host copy is stale
  void clear() { host_->clear(); hostValid_ = true; devValid_ = false; devN_ = 0; }
  // pcl::removeNaNFromPointCloud(c, c, idx) on a caller-filled host cloud (only clouds flagged !is_dense are touched)
  void dropNonFinite();
  // exchange contents with another cloud of the same context (the reference swaps cloud pointers)
  void swap(DualCloud& o);

 private:
  Cloud::Ptr host_;
  Context* ctx_;
  int slot_;
  bool hostValid_, devValid_;
  int devN_;
  std::vector<float> buf_;
};

// pcl::PointXYZI (32 B) <-> packed float4 (16 B)
inline void pack(const Cloud& c, std::vector<float>& out) {
  out.resize(c.points.size() * 4);
  for (std::size_t i = 0; i < c.points.size(); i++) {
    out[4 * i + 0] = c.points[i].x;
    out[4 * i + 1] = c.points[i].y;
    out[4 * i + 2] = c.points[i].z;
    out[4 * i + 3] = c.points[i].intensity;
  }
}
inline void unpack(const float* p, std::size_t n, Cloud& c) {
  c.points.resize(n);
  for (std::size_t i = 0; i < n; i++) {
    c.points[i].x = p[4 * i + 0];
    c.points[i].y = p[4 * i + 1];
    c.points[i].z = p[4 * i + 2];
    c.points[i].intensity = p[4 * i + 3];
  }
  c.width = static_cast<std::uint32_t>(n);
  c.height = 1;
  c.is_dense = true;
}

inline float leafOf(const pcl::VoxelGrid<pcl::PointXYZI>& f) {
#ifdef LOAM_B200_COMPAT_PCL
  return f.leafX();
#else
  return f.getLeafSize()[0];
#endif
}

inline void fillPose(const Twist& t, loam_b200_pose& p) {
  p.rot[0] = t.rot_x.rad(); p.rot[1] = t.rot_y.rad(); p.rot[2] = t.rot_z.rad();
  p.sin_[0] = t.rot_x.sin(); p.sin_[1] = t.rot_y.sin(); p.sin_[2] = t.rot_z.sin();
  p.cos_[0] = t.rot_x.cos(); p.cos_[1] = t.rot_y.cos(); p.cos_[2] = t.rot_z.cos();
  p.pos[0] = t.pos.x(); p.pos[1] = t.pos.y(); p.pos[2] = t.pos.z();
}

// Solve + degeneracy handling shared by odometry and mapping (BasicLaserOdometry.cpp:559-597,
// BasicLaserMapping.cpp:867-905): x = colPivHouseholderQr(AtA).solve(AtB); on the first iteration the eigenvalues of
// AtA below `eigenThreshold` (ascending, stop at the first that is not) zero ROWS of the eigenvector matrix copy and
// P = V^-1 * V2; degenerate -> x = P x.
struct GaussNewtonSolver {
  bool isDegenerate = false;
  float P[36];  // row-major
  void solve(const loam_b200_normal_eq& ne, bool firstIteration, float eigenThreshold, float x[6]);
};

// LOAM_B200_DEVICE_LOOP=1 (read once per process) runs the Gauss-Newton loops through loam_b200_odom_solve /
// loam_b200_map_solve: pose kept on the device, the whole loop one launch of a CUDA graph with a WHILE node
// (csrc/lmstep.cuh, loam_b200.cu), one host round trip per loop.  Unset or any other value: one iteration kernel and
// one host solve per iteration (the default).
bool deviceResidentLoops();

// host-side pcl::VoxelGrid replacement: one GPU call
void voxelFilter(Context& ctx, const Cloud& in, float leaf, Cloud& out, std::vector<float>& scratchIn,
                 std::vector<float>& scratchOut);

}  // namespace b200
}  // namespace loam
