// Device pcl::VoxelGrid<PointXYZI> (centroid of all fields per occupied voxel, output in ascending voxel index).
// Semantics follow PCL's published applyFilter (bbox -> min_b/div_b -> linear voxel index -> sort -> run means,
// "leaf size too small" guard returns the input); call sites in the reference: BasicLaserMapping.cpp:519-527
// (feature stacks, 0.2 / 0.4 m) and :580-588 (per-cube map maintenance).  Runs are averaged in (voxel, input order).
#pragma once

#include "lbvh.cuh"

namespace loamb {

// defined in loam_b200.cu: LSD radix sort of (keys_a, vals_a) in c->sort; sorted arrays returned through the out params
int radix_sort_pairs(loam_b200_ctx* c, int m, int key_bits, unsigned** keys_out = nullptr, int** vals_out = nullptr,
                     const int* n_dev = nullptr);

// heads[i] = 1 when sorted key i starts a run; per-block totals for the scan (32-bit voxel keys; 64-bit keys of the
// whole-run map, densemap.cuh)
constexpr int SCAN_BS = 1024;
template <typename K>
__global__ void __launch_bounds__(SCAN_BS)
voxel_head_kernel(const K* __restrict__ keys, int n, unsigned* __restrict__ pos, unsigned* __restrict__ block_sums) {
  __shared__ unsigned ws[32];
  const int i = blockIdx.x * SCAN_BS + threadIdx.x;
  const unsigned h = (i < n && (i == 0 || keys[i] != keys[i - 1])) ? 1u : 0u;
  unsigned x = h;
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned y = __shfl_up_sync(0xffffffffu, x, o);
    if ((threadIdx.x & 31) >= o) x += y;
  }
  if ((threadIdx.x & 31) == 31) ws[threadIdx.x >> 5] = x;
  __syncthreads();
  if (threadIdx.x < 32) {
    unsigned w = ws[threadIdx.x];
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned y = __shfl_up_sync(0xffffffffu, w, o);
      if (threadIdx.x >= o) w += y;
    }
    ws[threadIdx.x] = w;
  }
  __syncthreads();
  const unsigned incl = x + ((threadIdx.x >> 5) ? ws[(threadIdx.x >> 5) - 1] : 0u);
  if (i < n) pos[i] = (incl - h) | (h << 31);  // exclusive rank inside the block + head flag
  if (threadIdx.x == SCAN_BS - 1) block_sums[blockIdx.x] = incl;
}

// one thread per run head: mean of x, y, z, intensity over the run, in sorted order
__global__ void voxel_centroid_kernel(const float4* __restrict__ p, const unsigned* __restrict__ keys,
                                      const int* __restrict__ vals, const unsigned* __restrict__ pos,
                                      const unsigned* __restrict__ block_off, int n, float4* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const unsigned pv = pos[i];
  if (!(pv >> 31)) return;
  const unsigned dst = (pv & 0x7fffffffu) + block_off[i / SCAN_BS];
  const unsigned k = keys[i];
  float sx = 0.f, sy = 0.f, sz = 0.f, si = 0.f;
  int cnt = 0;
  for (int u = i; u < n && keys[u] == k; u++) {
    const float4 q = p[vals[u]];
    sx += q.x; sy += q.y; sz += q.z; si += q.w;
    cnt++;
  }
  const float fn = (float)cnt;
  out[dst] = make_float4(sx / fn, sy / fn, sz / fn, si / fn);
}

struct VoxMeta {
  int minb0, minb1, minb2, div0, div1, overflow;
};

// bbox -> voxel grid origin / extents on the device (pcl::VoxelGrid::applyFilter's min_b_ / div_b_ and its int32
// overflow guard "Leaf size is too small for the input dataset")
__device__ __forceinline__ VoxMeta voxel_meta_from_bbox(const float* mn, const float* mx, float inv) {
  const long long dx = (long long)((mx[0] - mn[0]) * inv) + 1, dy = (long long)((mx[1] - mn[1]) * inv) + 1,
                  dz = (long long)((mx[2] - mn[2]) * inv) + 1;
  VoxMeta m;
  m.overflow = (dx * dy * dz > 2147483647ll) ? 1 : 0;
  m.minb0 = (int)floorf(mn[0] * inv);
  m.minb1 = (int)floorf(mn[1] * inv);
  m.minb2 = (int)floorf(mn[2] * inv);
  m.div0 = (int)floorf(mx[0] * inv) - m.minb0 + 1;
  m.div1 = (int)floorf(mx[1] * inv) - m.minb1 + 1;
  return m;
}

// on overflow every point keeps its own key (= its index), which makes the filter an identity exactly like pcl's
// early return.  The guard bounds the truncated extents, not the div product, so keys can pass 2^31: pcl's int32 key
// wraps there, which is computed in unsigned arithmetic (same bits, no signed overflow).
__device__ __forceinline__ unsigned voxel_key_of(const float4& q, float inv, const VoxMeta& m, int i) {
  if (m.overflow) return (unsigned)i;
  const int i0 = (int)(floorf(q.x * inv) - (float)m.minb0);
  const int i1 = (int)(floorf(q.y * inv) - (float)m.minb1);
  const int i2 = (int)(floorf(q.z * inv) - (float)m.minb2);
  return (unsigned)i0 + (unsigned)i1 * (unsigned)m.div0 + (unsigned)i2 * (unsigned)m.div0 * (unsigned)m.div1;
}

__global__ void voxel_meta_kernel(const unsigned* __restrict__ bb, float inv, VoxMeta* __restrict__ meta) {
  if (threadIdx.x != 0) return;
  float mn[3], mx[3];
  for (int a = 0; a < 3; a++) { mn[a] = dec_f(bb[a]); mx[a] = dec_f(bb[3 + a]); }
  *meta = voxel_meta_from_bbox(mn, mx, inv);
}

__global__ void voxel_key_meta_kernel(const float4* __restrict__ p, int n, float inv, const VoxMeta* __restrict__ meta,
                                      unsigned* __restrict__ keys, int* __restrict__ vals) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const VoxMeta m = *meta;
  vals[i] = i;
  keys[i] = voxel_key_of(p[i], inv, m, i);
}

// defined in loam_b200.cu: the single-launch cluster filter of clustersort.cuh (n <= CS_MAX_N); roundtrip = optional
// MapIterArgs* of the to-map-and-back transform applied to the input first (d_tmp then receives the transformed cloud)
int voxel_filter_cluster(loam_b200_ctx* c, const float4* d_in, int n, float leaf, const void* roundtrip, float4* d_tmp,
                         float4* d_out, int* d_count);
bool cluster_path_ok(const loam_b200_ctx* c, int n);

inline int voxel_grid_async(loam_b200_ctx* c, const float4* d_in, int n, float leaf, float4* d_out, int* d_count) {
  if (n <= 0) {
    LB_CUDA(c, cudaMemsetAsync(d_count, 0, sizeof(int), c->stream));
    return LOAM_B200_OK;
  }
  if (cluster_path_ok(c, n)) return voxel_filter_cluster(c, d_in, n, leaf, nullptr, nullptr, d_out, d_count);
  SortScratch& s = c->sort;
  LB_CUDA(c, s.keys_a.reserve(n));
  LB_CUDA(c, s.keys_b.reserve(n));
  LB_CUDA(c, s.vals_a.reserve(n));
  LB_CUDA(c, s.vals_b.reserve(n));
  LB_CUDA(c, c->bbox.reserve(16));
  unsigned* bb = reinterpret_cast<unsigned*>(c->bbox.p);
  VoxMeta* meta = reinterpret_cast<VoxMeta*>(c->bbox.p + 8);
  const float inv = 1.0f / leaf;
  bbox_init_kernel<<<1, 32, 0, c->stream>>>(bb);
  LB_LAUNCH_CHECK(c);
  const int bbox_blocks = std::min((n + 255) / 256, c->sm_count * 2);
  bbox_kernel<<<bbox_blocks, 256, 0, c->stream>>>(d_in, n, bb);
  LB_LAUNCH_CHECK(c);
  voxel_meta_kernel<<<1, 32, 0, c->stream>>>(bb, inv, meta);
  LB_LAUNCH_CHECK(c);
  voxel_key_meta_kernel<<<(n + 255) / 256, 256, 0, c->stream>>>(d_in, n, inv, meta, s.keys_a.p, s.vals_a.p);
  LB_LAUNCH_CHECK(c);
  // voxel indices are < 2^31 by pcl's own guard: four 8-bit passes
  unsigned* ka = nullptr;
  int* va = nullptr;
  {
    const int rc = radix_sort_pairs(c, n, 32, &ka, &va);
    if (rc) return rc;
  }
  const int nb = (n + SCAN_BS - 1) / SCAN_BS;
  LB_CUDA(c, c->vox_key.reserve((size_t)n + nb + 8));
  unsigned* pos = c->vox_key.p;
  unsigned* bsum = c->vox_key.p + n;
  voxel_head_kernel<<<nb, SCAN_BS, 0, c->stream>>>(ka, n, pos, bsum);
  LB_LAUNCH_CHECK(c);
  radix_scan_kernel<<<1, 1024, 0, c->stream>>>(bsum, nb + 1, d_count);  // entry nb = number of voxels, mirrored to d_count
  LB_LAUNCH_CHECK(c);
  voxel_centroid_kernel<<<(n + 255) / 256, 256, 0, c->stream>>>(d_in, ka, va, pos, bsum, n, d_out);
  LB_LAUNCH_CHECK(c);
  return LOAM_B200_OK;
}

// synchronous convenience: *count on the host
inline int voxel_grid_device(loam_b200_ctx* c, const float4* d_in, int n, float leaf, float4* d_out, int* count) {
  *count = 0;
  if (n <= 0) return LOAM_B200_OK;
  LB_CUDA(c, c->dcount.reserve(512));  // one allocation for every stage counter (stages.inc: D_NUM)
  int rc = voxel_grid_async(c, d_in, n, leaf, d_out, c->dcount.p + 63);
  if (rc) return rc;
  LB_CUDA(c, cudaMemcpyAsync(count, c->dcount.p + 63, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
  LB_CUDA(c, cudaStreamSynchronize(c->stream));
  return LOAM_B200_OK;
}

}  // namespace loamb
