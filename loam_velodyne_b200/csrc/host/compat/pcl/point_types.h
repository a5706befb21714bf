// Minimal PCL point types for builds without PCL (the ROS adapters upstream compile against the real library;
// in that case put the real PCL include directory first and drop compat/ from the include path).
// Layout matches PCL: PointXYZ is 16 B, PointXYZI 32 B with intensity at byte 16, PointXYZINormal 48 B with the normal
// at byte 16, intensity at 32 and curvature at 36, all 16 B aligned.
#pragma once
#include <cmath>

#ifndef pcl_isfinite
#define pcl_isfinite(x) std::isfinite(x)
#endif

namespace pcl {

struct alignas(16) PointXYZ {
  union {
    float data[4];
    struct { float x, y, z; };
  };
  PointXYZ() { data[0] = data[1] = data[2] = 0.f; data[3] = 1.f; }
  PointXYZ(float px, float py, float pz) { data[0] = px; data[1] = py; data[2] = pz; data[3] = 1.f; }
};

struct alignas(16) PointXYZI {
  union {
    float data[4];
    struct { float x, y, z; };
  };
  union {
    struct { float intensity; };
    float data_c[4];
  };
  PointXYZI() {
    data[0] = data[1] = data[2] = 0.f; data[3] = 1.f;
    data_c[0] = data_c[1] = data_c[2] = data_c[3] = 0.f;
  }
};

// 48 B: xyz + pad, normal_x/y/z + pad, intensity, curvature, 2 pad
struct alignas(16) PointXYZINormal {
  union {
    float data[4];
    struct { float x, y, z; };
  };
  union {
    float data_n[4];
    float normal[3];
    struct { float normal_x, normal_y, normal_z; };
  };
  union {
    struct { float intensity; float curvature; };
    float data_c[4];
  };
  PointXYZINormal() {
    data[0] = data[1] = data[2] = 0.f; data[3] = 1.f;
    data_n[0] = data_n[1] = data_n[2] = data_n[3] = 0.f;
    data_c[0] = data_c[1] = data_c[2] = data_c[3] = 0.f;
  }
};
static_assert(sizeof(PointXYZINormal) == 48, "PCL's PointXYZINormal layout");

}  // namespace pcl
