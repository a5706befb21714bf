// Small-cloud building blocks that live entirely inside ONE thread-block cluster (16 CTAs, distributed shared memory).
//
// The feature stacks of a sweep (5 k corner / 20 k surface points) and the odometry's last-sweep clouds are far too
// small to fill the GPU, and as chains of 12-14 tiny launches (bbox, keys, histogram, four radix passes, heads, scan,
// centroids / gather, leaves, Karras, refit) they were bound by the host's launch rate, not by the GPU.  Here the
// (key, index) pairs of such a cloud stay in the shared memory of the cluster's CTAs for the whole
// LSD sort: per 8-bit digit every CTA ranks its tile (match.any, stable), the eight per-CTA digit counts are exchanged
// through DSMEM around one cluster barrier, and the pairs are scattered straight into the destination CTA's shared
// memory (st.shared::cluster).  The surrounding steps (bounding box, keys, run heads + centroids, or gather + leaves +
// Karras + refit) are phases of the same launch, separated by cluster barriers.
//   voxel_filter_cluster_kernel : pcl::VoxelGrid (optionally preceded by the mapping stage's to-map-and-back transform)
//   bvh_build_cluster_kernel    : the whole LBVH build of lbvh.cuh
// Clouds above CS_MAX_N points take the multi-launch path (onesweep sort over HBM).
#pragma once

#include <cooperative_groups.h>

#include "lbvh.cuh"
#include "mapping_lm.cuh"
#include "voxel.cuh"

namespace loamb {

namespace cg = cooperative_groups;

#ifndef LOAM_B200_CS_CL
#define LOAM_B200_CS_CL 16                // CTAs per cluster (8 = portable maximum; 16 = non-portable opt-in, supported by H100)
#endif
#ifndef LOAM_B200_CS_THREADS
#define LOAM_B200_CS_THREADS 512
#endif
constexpr int CS_CL = LOAM_B200_CS_CL;
constexpr int CS_THREADS = LOAM_B200_CS_THREADS;
constexpr int CS_NW = CS_THREADS / 32;
constexpr int CS_CAP = 8192;              // pairs per CTA
constexpr int CS_MAX_N = CS_CL * CS_CAP;  // 131072 with 16 CTAs

struct ClusterSortSmem {
  unsigned keys[2][CS_CAP];
  int vals[2][CS_CAP];
  unsigned short rank[CS_CAP];
  unsigned wcount[CS_NW][256];
  unsigned cta_cnt[256];  // this CTA's digit counts, read by the other CTAs of the cluster
  unsigned gbase[256];
  unsigned wsum[CS_NW];
  unsigned scal[4];       // per-CTA scalars exchanged across the cluster (e.g. number of run heads)
  float bb[6];            // this CTA's bounding box
  float gbb[6];           // the cloud's bounding box
};

// element g of the cluster-distributed array lives in CTA g / per at offset g % per
__device__ __forceinline__ int cs_local_count(int n, int per, unsigned rank) {
  return max(0, min(per, n - (int)rank * per));
}

// LSD radix sort of the distributed (key, val) pairs held in sm.keys[0] / sm.vals[0]; returns the buffer (0 / 1) that
// holds the sorted pairs.  Passes whose digit is identical for every key are skipped.  All threads of all CTAs call it.
__device__ __forceinline__ int cluster_sort(ClusterSortSmem& sm, int n, int per, int passes) {
  cg::cluster_group cluster = cg::this_cluster();
  const unsigned my = cluster.block_rank();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int m_local = cs_local_count(n, per, my);
  const int pw = (((per + CS_NW - 1) / CS_NW) + 31) & ~31;  // consecutive pairs owned by one warp
  const int wb = min(warp * pw, m_local), we = min(wb + pw, m_local);
  int cur = 0;
  for (int p = 0; p < passes; p++) {
    const int shift = 8 * p;
    for (int d = lane; d < 256; d += 32) sm.wcount[warp][d] = 0;
    __syncwarp();
    for (int i0 = wb; i0 < we; i0 += 32) {
      const int i = i0 + lane;
      const bool valid = i < we;
      const unsigned d = valid ? ((sm.keys[cur][i] >> shift) & 255u) : 256u;  // invalid lanes only match each other
      const unsigned peers = __match_any_sync(0xffffffffu, d);
      const unsigned before = __popc(peers & ((1u << lane) - 1u));
      unsigned prior = 0;
      if (valid) {
        prior = sm.wcount[warp][d];
        sm.rank[i] = (unsigned short)(prior + before);
      }
      __syncwarp();
      if (valid && before == 0) sm.wcount[warp][d] = prior + __popc(peers);
      __syncwarp();
    }
    __syncthreads();
    if (threadIdx.x < 256) {
      unsigned acc = 0;
#pragma unroll
      for (int wv = 0; wv < CS_NW; wv++) {
        const unsigned c = sm.wcount[wv][threadIdx.x];
        sm.wcount[wv][threadIdx.x] = acc;
        acc += c;
      }
      sm.cta_cnt[threadIdx.x] = acc;
    }
    cluster.sync();
    unsigned tot = 0, below = 0;
    if (threadIdx.x < 256) {
#pragma unroll
      for (unsigned r = 0; r < CS_CL; r++) {
        const unsigned c = cluster.map_shared_rank(&sm.cta_cnt[0], r)[threadIdx.x];
        if (r < my) below += c;
        tot += c;
      }
    }
    unsigned x = tot;
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned y = __shfl_up_sync(0xffffffffu, x, o);
      if (lane >= o) x += y;
    }
    if (lane == 31) sm.wsum[warp] = x;
    const int uniform = __syncthreads_or(threadIdx.x < 256 && tot == (unsigned)n);  // same verdict in every CTA
    if (threadIdx.x < 256) {
      unsigned woff = 0;
      for (int w = 0; w < warp; w++) woff += sm.wsum[w];
      sm.gbase[threadIdx.x] = (x - tot) + woff + below;
    }
    __syncthreads();
    if (!uniform) {
      for (int i0 = wb; i0 < we; i0 += 32) {
        const int i = i0 + lane;
        if (i < we) {
          const unsigned k = sm.keys[cur][i];
          const unsigned d = (k >> shift) & 255u;
          const unsigned g = sm.gbase[d] + sm.wcount[warp][d] + sm.rank[i];
          const unsigned dest = g / (unsigned)per, off = g - dest * (unsigned)per;
          cluster.map_shared_rank(&sm.keys[cur ^ 1][0], dest)[off] = k;
          cluster.map_shared_rank(&sm.vals[cur ^ 1][0], dest)[off] = sm.vals[cur][i];
        }
      }
    }
    cluster.sync();
    if (!uniform) cur ^= 1;
  }
  return cur;
}

// bounding box of the cloud: per-CTA partial -> DSMEM exchange -> sm.gbb (identical in every CTA)
__device__ __forceinline__ void cluster_bbox(ClusterSortSmem& sm, float mn[3], float mx[3]) {
  cg::cluster_group cluster = cg::this_cluster();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float* wred = reinterpret_cast<float*>(&sm.wcount[0][0]);  // [CS_NW][6], free before the sort starts
#pragma unroll
  for (int a = 0; a < 3; a++) {
    for (int o = 16; o > 0; o >>= 1) {
      mn[a] = fminf(mn[a], __shfl_xor_sync(0xffffffffu, mn[a], o));
      mx[a] = fmaxf(mx[a], __shfl_xor_sync(0xffffffffu, mx[a], o));
    }
    if (lane == 0) {
      wred[warp * 6 + a] = mn[a];
      wred[warp * 6 + 3 + a] = mx[a];
    }
  }
  __syncthreads();
  if (threadIdx.x < 6) {
    float v = wred[threadIdx.x];
    for (int w = 1; w < CS_NW; w++)
      v = threadIdx.x < 3 ? fminf(v, wred[w * 6 + threadIdx.x]) : fmaxf(v, wred[w * 6 + threadIdx.x]);
    sm.bb[threadIdx.x] = v;
  }
  cluster.sync();
  if (threadIdx.x < 6) {
    float v = cluster.map_shared_rank(&sm.bb[0], 0)[threadIdx.x];
    for (unsigned r = 1; r < CS_CL; r++) {
      const float o = cluster.map_shared_rank(&sm.bb[0], r)[threadIdx.x];
      v = threadIdx.x < 3 ? fminf(v, o) : fmaxf(v, o);
    }
    sm.gbb[threadIdx.x] = v;
  }
  __syncthreads();
}

// pcl::VoxelGrid of in[0..n) -> out, number of voxels -> *count_out.  ROUNDTRIP: every input point first goes through
// pointAssociateToMap / pointAssociateTobeMapped with the predicted pose (stack_roundtrip_kernel's arithmetic); the
// transformed cloud is kept in tmp.  One cluster = the whole launch.
template <bool ROUNDTRIP>
__global__ void __cluster_dims__(CS_CL, 1, 1) __launch_bounds__(CS_THREADS)
voxel_filter_cluster_kernel(const float4* __restrict__ in, int n, float inv, MapIterArgs a, float4* __restrict__ tmp,
                            float4* __restrict__ out, int* __restrict__ count_out) {
  extern __shared__ __align__(16) unsigned char cs_raw[];
  ClusterSortSmem& sm = *reinterpret_cast<ClusterSortSmem*>(cs_raw);
  cg::cluster_group cluster = cg::this_cluster();
  const unsigned my = cluster.block_rank();
  const int per = (n + CS_CL - 1) / CS_CL;
  const int m_local = cs_local_count(n, per, my);
  const int g0 = (int)my * per;
  const float4* pts = ROUNDTRIP ? tmp : in;

  float mn[3] = {FLT_MAX, FLT_MAX, FLT_MAX}, mx[3] = {-FLT_MAX, -FLT_MAX, -FLT_MAX};
  for (int i = threadIdx.x; i < m_local; i += CS_THREADS) {
    float4 q = in[g0 + i];
    if (ROUNDTRIP) {
      q = stack_roundtrip(a, q);
      tmp[g0 + i] = q;
    }
    mn[0] = fminf(mn[0], q.x); mx[0] = fmaxf(mx[0], q.x);
    mn[1] = fminf(mn[1], q.y); mx[1] = fmaxf(mx[1], q.y);
    mn[2] = fminf(mn[2], q.z); mx[2] = fmaxf(mx[2], q.z);
  }
  cluster_bbox(sm, mn, mx);
  const VoxMeta vm = voxel_meta_from_bbox(sm.gbb, sm.gbb + 3, inv);
  for (int i = threadIdx.x; i < m_local; i += CS_THREADS) {
    const float4 q = ROUNDTRIP ? tmp[g0 + i] : in[g0 + i];  // own earlier write when ROUNDTRIP
    sm.keys[0][i] = voxel_key_of(q, inv, vm, g0 + i);
    sm.vals[0][i] = g0 + i;
  }
  __syncthreads();
  const int cur = cluster_sort(sm, n, per, 4);

  // run heads: position of every head inside this CTA (block scan in rounds, no global traffic) -> exchange the CTA
  // totals -> centroids.  The positions live in the sort's spare value buffer.
  auto key_at = [&](int g) -> unsigned {
    const int r = g / per;
    return cluster.map_shared_rank(&sm.keys[cur][0], r)[g - r * per];
  };
  int* head_pos = &sm.vals[cur ^ 1][0];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  unsigned carry = 0;
  for (int base = 0; base < m_local; base += CS_THREADS) {
    const int i = base + threadIdx.x;
    const bool head = i < m_local && (g0 + i == 0 || sm.keys[cur][i] != (i > 0 ? sm.keys[cur][i - 1] : key_at(g0 - 1)));
    const unsigned bal = __ballot_sync(0xffffffffu, head);
    if (lane == 0) sm.wsum[warp] = __popc(bal);
    __syncthreads();
    unsigned woff = 0, round_total = 0;
    for (int w = 0; w < CS_NW; w++) {
      const unsigned c = sm.wsum[w];
      if (w < warp) woff += c;
      round_total += c;
    }
    if (i < m_local) head_pos[i] = head ? (int)(carry + woff + __popc(bal & ((1u << lane) - 1u))) : -1;
    carry += round_total;
    __syncthreads();
  }
  if (threadIdx.x == 0) sm.scal[0] = carry;
  cluster.sync();
  unsigned cta_base = 0, total = 0;
  for (unsigned r = 0; r < CS_CL; r++) {
    const unsigned h = cluster.map_shared_rank(&sm.scal[0], r)[0];
    if (r < my) cta_base += h;
    total += h;
  }
  if (my == 0 && threadIdx.x == 0) *count_out = (int)total;
  // centroids: every thread walks the runs that start at its elements, no barrier in between (the walk is a chain of
  // dependent loads; with a barrier per round the slowest run of each round set the pace)
  for (int i = threadIdx.x; i < m_local; i += CS_THREADS) {
    const int hp = head_pos[i];
    if (hp < 0) continue;
    const unsigned k = sm.keys[cur][i];
    float sx = 0.f, sy = 0.f, sz = 0.f, si = 0.f;
    int cnt = 0;
    // the run may continue in the next CTAs' shared memory
    unsigned r = my;
    int off = i;
    const unsigned* kp = &sm.keys[cur][0];
    const int* vp = &sm.vals[cur][0];
    for (int g = g0 + i; g < n; g++) {
      if (kp[off] != k) break;
      const float4 q = __ldcg(&pts[vp[off]]);
      sx += q.x; sy += q.y; sz += q.z; si += q.w;
      cnt++;
      if (++off == per) {
        off = 0;
        r++;
        if (r < CS_CL) {
          kp = cluster.map_shared_rank(&sm.keys[cur][0], r);
          vp = cluster.map_shared_rank(&sm.vals[cur][0], r);
        }
      }
    }
    const float fn = (float)cnt;
    out[cta_base + (unsigned)hp] = make_float4(sx / fn, sy / fn, sz / fn, si / fn);
  }
  cluster.sync();  // nobody leaves while a neighbour may still read its shared memory
}

// generic (key, value) sort of a small array, in place allowed (everything is loaded before anything is stored)
__global__ void __cluster_dims__(CS_CL, 1, 1) __launch_bounds__(CS_THREADS)
cluster_sort_pairs_kernel(const unsigned* keys_in, const int* vals_in, int n, const int* __restrict__ n_dev, int passes,
                          unsigned* keys_out, int* vals_out) {
  extern __shared__ __align__(16) unsigned char cs_raw[];
  ClusterSortSmem& sm = *reinterpret_cast<ClusterSortSmem*>(cs_raw);
  cg::cluster_group cluster = cg::this_cluster();
  if (n_dev) n = min(n, *n_dev);
  if (n <= 0) return;  // uniform over the cluster
  const unsigned my = cluster.block_rank();
  const int per = (n + CS_CL - 1) / CS_CL;
  const int m_local = cs_local_count(n, per, my);
  const int g0 = (int)my * per;
  for (int i = threadIdx.x; i < m_local; i += CS_THREADS) {
    sm.keys[0][i] = keys_in[g0 + i];
    sm.vals[0][i] = vals_in[g0 + i];
  }
  __syncthreads();
  const int cur = cluster_sort(sm, n, per, passes);
  for (int i = threadIdx.x; i < m_local; i += CS_THREADS) {
    keys_out[g0 + i] = sm.keys[cur][i];
    vals_out[g0 + i] = sm.vals[cur][i];
  }
  cluster.sync();
}

// LBVH build of lbvh.cuh in one launch: bbox -> Morton keys -> cluster sort -> gather -> leaves -> Karras -> refit
// One launch builds up to TWO trees (one cluster each: the last corner / last surface cloud of the odometry stage are
// rebuilt together every sweep); a1.n == 0 with a grid of one cluster builds one.
struct BvhBuildArgs {
  const float4* pts;
  int n, n_leaf;
  float4* sorted;
  unsigned* leaf_key;
  BvhNode* nodes;
  int* parent;
  float4* box_lo;
  float4* box_hi;
  int* flags;
};
__global__ void __cluster_dims__(CS_CL, 1, 1) __launch_bounds__(CS_THREADS)
bvh_build_cluster_kernel(BvhBuildArgs a0, BvhBuildArgs a1) {
  const BvhBuildArgs& A = blockIdx.x < CS_CL ? a0 : a1;
  const float4* __restrict__ pts = A.pts;
  const int n = A.n, n_leaf = A.n_leaf;
  if (n <= 0) return;  // the whole cluster leaves together
  float4* __restrict__ sorted = A.sorted;
  unsigned* __restrict__ leaf_key = A.leaf_key;
  BvhNode* __restrict__ nodes = A.nodes;
  int* __restrict__ parent = A.parent;
  float4* __restrict__ box_lo = A.box_lo;
  float4* __restrict__ box_hi = A.box_hi;
  int* __restrict__ flags = A.flags;
  extern __shared__ __align__(16) unsigned char cs_raw[];
  ClusterSortSmem& sm = *reinterpret_cast<ClusterSortSmem*>(cs_raw);
  cg::cluster_group cluster = cg::this_cluster();
  const unsigned my = cluster.block_rank();
  const int per = (n + CS_CL - 1) / CS_CL;
  const int m_local = cs_local_count(n, per, my);
  const int g0 = (int)my * per;

  float mn[3] = {FLT_MAX, FLT_MAX, FLT_MAX}, mx[3] = {-FLT_MAX, -FLT_MAX, -FLT_MAX};
  for (int i = threadIdx.x; i < m_local; i += CS_THREADS) {
    const float4 q = pts[g0 + i];
    mn[0] = fminf(mn[0], q.x); mx[0] = fmaxf(mx[0], q.x);
    mn[1] = fminf(mn[1], q.y); mx[1] = fmaxf(mx[1], q.y);
    mn[2] = fminf(mn[2], q.z); mx[2] = fmaxf(mx[2], q.z);
  }
  cluster_bbox(sm, mn, mx);
  for (int i = threadIdx.x; i < m_local; i += CS_THREADS) {
    sm.keys[0][i] = morton_key(pts[g0 + i], sm.gbb[0], sm.gbb[1], sm.gbb[2], sm.gbb[3], sm.gbb[4], sm.gbb[5]);
    sm.vals[0][i] = g0 + i;
  }
  __syncthreads();
  const int cur = cluster_sort(sm, n, per, 4);
  for (int i = threadIdx.x; i < m_local; i += CS_THREADS) {
    const int g = g0 + i, o = sm.vals[cur][i];
    float4 p = pts[o];
    p.w = __int_as_float(o);
    sorted[g] = p;
    if (g % LEAF_SIZE == 0) leaf_key[g / LEAF_SIZE] = sm.keys[cur][i];
  }
  __threadfence();
  cluster.sync();
  const int ctid = (int)my * CS_THREADS + threadIdx.x, cthreads = CS_CL * CS_THREADS;
  for (int l = ctid; l < n_leaf; l += cthreads) leaf_body(l, sorted, n, n_leaf, box_lo, box_hi, flags);
  if (n_leaf > 1) {
    for (int i = ctid; i < n_leaf - 1; i += cthreads) karras_body(i, leaf_key, n_leaf, nodes, parent);
    __threadfence();
    cluster.sync();
    for (int l = ctid; l < n_leaf; l += cthreads) refit_body(l, n_leaf, nodes, parent, box_lo, box_hi, flags);
  }
  cluster.sync();
}

}  // namespace loamb
