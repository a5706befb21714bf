// Fixed-radius exact 5-NN for the scan-to-map loop.
//
// The reference only uses a map correspondence when the 5th neighbour is closer than 1 m
// (pointSearchSqDis[4] < 1.0, BasicLaserMapping.cpp:671,760), so the search is a fixed-radius query: every accepted
// neighbour lies in the 3 x 3 x 3 block of 1 m cells around the query.  The BVH walk on this workload makes ~48
// dependent node visits per query with few active lanes;
// a Morton-free uniform grid removes both the dependency chain and the divergence:
//   build : cell key (z, y, x) per point -> LSD radix sort -> points gathered in cell order (xyz + original index) ->
//           open-addressing table cell -> (start, count)
//   query : 27 independent table probes (issued nine at a time), then the candidates of each occupied cell, four
//           loads in flight; a candidate enters the running top-5 only when strictly closer than the current 5th
//           (nanoflann's KNNResultSet::addPoint, nanoflann.hpp:115-139), distances accumulate x -> y -> z in fp32
//           exactly like L2_Simple_Adaptor::evalMetric (nanoflann.hpp:372-379).
// Cell coordinates are floorf(x) - origin with an INTEGER origin, so |p - q| < 1 implies the two cell indices differ
// by at most one per axis exactly (no subtraction rounding) and the 27-cell candidate set is a true superset.
// The general-radius searches (odometry 1-NN within 5 m, loam_b200_tree_knn) keep the BVH of lbvh.cuh.
#pragma once

#include "lbvh.cuh"
#include "shard.cuh"

namespace loamb {

struct GridMeta {       // written by grid_meta_kernel, read by every later kernel (no host round trip)
  int ox, oy, oz;       // integer origin = floor(bbox min) - 1
  int nx, ny, nz;       // cells per axis (clamped so the key fits 31 bits)
};

struct GridView {
  const uint4* table;   // {key + 1 (0 = empty), start, count, -}
  unsigned mask;        // table size - 1 (power of two)
  const float4* sorted; // points in cell order, w = original index bits
  const GridMeta* meta;
  int m;                // upper bound of the point count (0 = empty grid)
};

__device__ __forceinline__ unsigned grid_hash(unsigned k) {
  k ^= k >> 16;
  k *= 0x7feb352dU;
  k ^= k >> 15;
  k *= 0x846ca68bU;
  k ^= k >> 16;
  return k;
}

__global__ void grid_meta_kernel(const unsigned* __restrict__ bb, GridMeta* __restrict__ meta) {
  if (threadIdx.x != 0) return;
  const float lx = dec_f(bb[0]), ly = dec_f(bb[1]), lz = dec_f(bb[2]);
  const float hx = dec_f(bb[3]), hy = dec_f(bb[4]), hz = dec_f(bb[5]);
  GridMeta g;
  g.ox = (int)floorf(lx) - 1;
  g.oy = (int)floorf(ly) - 1;
  g.oz = (int)floorf(lz) - 1;
  g.nx = min(max((int)floorf(hx) - g.ox + 2, 1), 1290);
  g.ny = min(max((int)floorf(hy) - g.oy + 2, 1), 1290);
  g.nz = min(max((int)floorf(hz) - g.oz + 2, 1), 1290);
  *meta = g;
}

__device__ __forceinline__ unsigned grid_key(const GridMeta& g, int cx, int cy, int cz) {
  return (unsigned)((cz * g.ny + cy) * g.nx + cx);
}

__global__ void grid_key_kernel(const float4* __restrict__ p, int m, const GridMeta* __restrict__ meta,
                                unsigned* __restrict__ keys, int* __restrict__ vals,
                                const int* __restrict__ n_dev = nullptr) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= m) return;
  if (n_dev && i >= *n_dev) {  // padding up to the launch bound sorts behind every real key
    keys[i] = 0xffffffffu;
    vals[i] = i;
    return;
  }
  const GridMeta g = *meta;
  const float4 q = p[i];
  const int cx = min(max((int)floorf(q.x) - g.ox, 0), g.nx - 1);
  const int cy = min(max((int)floorf(q.y) - g.oy, 0), g.ny - 1);
  const int cz = min(max((int)floorf(q.z) - g.oz, 0), g.nz - 1);
  keys[i] = grid_key(g, cx, cy, cz);
  vals[i] = i;
}

// one thread per sorted point; run heads insert (key, start, count) with linear probing
// n_cells (optional): receives the number of run heads = occupied cells (one atomic per block)
__global__ void grid_insert_kernel(const unsigned* __restrict__ keys, int m, uint4* __restrict__ table, unsigned mask,
                                   const int* __restrict__ n_dev = nullptr, int* __restrict__ n_cells = nullptr) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (n_dev) m = min(m, *n_dev);
  const bool head = i < m && (i == 0 || keys[i - 1] != keys[i]);
  if (n_cells) {
    const int heads = __syncthreads_count(head ? 1 : 0);
    if (threadIdx.x == 0 && heads > 0) atomicAdd(n_cells, heads);
  }
  if (!head) return;
  const unsigned k = keys[i];
  int cnt = 1;
  while (i + cnt < m && keys[i + cnt] == k) cnt++;
  unsigned h = grid_hash(k) & mask;
  for (unsigned tries = 0; tries <= mask; tries++) {  // bounded: a full table (cannot happen at load <= 0.5) must not hang the GPU
    const unsigned prev = atomicCAS(&table[h].x, 0u, k + 1u);
    if (prev == 0u) {
      table[h].y = (unsigned)i;
      table[h].z = (unsigned)cnt;
      return;
    }
    h = (h + 1) & mask;
  }
}

struct Top5 {
  float d[5], x[5], y[5], z[5];
  int idx[5];
};

// ---- eight lanes per query ------------------------------------------------------------------------------------
// The scan-to-map stage has only ~18 k queries per launch; one thread per query leaves ~4 warps per SM and the kernel
// was a serial latency chain.  Eight lanes share a query instead:
//   probe   : lane s looks up cells s, s+8, s+16, s+24 of the 3 x 3 x 3 block (all probes issued before any use);
//   balance : the 27 (start, count) pairs go to shared memory with an exclusive prefix of the counts, so the block's
//             candidates form ONE flattened list of T points; lane s takes candidates s, s+8, s+16, ... whatever cell
//             they come from (the first version let every lane walk its own cells: 8-9 of 32 lanes active in the
//             candidate loop because the centre cells hold most of the points);
//   merge   : each lane keeps a private top-5 (distance, position in the sorted cloud); five rounds of an 8-lane
//             shuffle arg-min ("take the smallest head, advance that lane") give the exact global top-5.
// Ties are broken by position in the sorted cloud (deterministic).
struct Cand5 {
  float d[5];
  int id[5];
};

__device__ __forceinline__ void cand5_offer(Cand5& r, float d, int id) {
  if (d < r.d[4]) {
    float cd = d;
    int ci = id;
#pragma unroll
    for (int s = 0; s < 5; s++) {
      if (cd < r.d[s]) {
        const float td = r.d[s];
        const int ti = r.id[s];
        r.d[s] = cd; r.id[s] = ci;
        cd = td; ci = ti;
      }
    }
  }
}

constexpr int GRID_SLOTS = 32;  // flattened cell slots per query: slot = lane * 4 + r (27 used)

// Can neighbour cell t = (dz + 1) * 9 + (dy + 1) * 3 + (dx + 1) of the 3 x 3 x 3 block hold a point closer than 1 m to a
// query whose position inside its own cell is (fx, fy, fz) in [0, 1)?  The nearest point of that cell is fx (1 - fx) away
// along an axis with offset -1 (+1).  On average 20.6 of the 27 cells pass (volume of the unit cube dilated by the unit
// ball), so a quarter of the table probes and candidate points is never touched.  The margin keeps every cell whose
// points could still evaluate to d^2 < 1 in fp32 (the comparison the search uses), so the result is unchanged.
// Measured: on the 20 M-point stress (HBM bound) the kernel gets 14 % faster; on the L2-resident 1 M map the saved loads
// do not pay for the extra instructions (10.1 M against 8.9 M warp instructions, 29.7 against 28.5 us), so the lookups
// carry a `prune` flag that the host sets for maps beyond L2 only.
__device__ __forceinline__ bool cell_in_reach(int t, float fx, float fy, float fz) {
  const int dx = t % 3 - 1, dy = (t / 3) % 3 - 1, dz = t / 9 - 1;
  const float ax = dx < 0 ? fx : (dx > 0 ? 1.f - fx : 0.f);
  const float ay = dy < 0 ? fy : (dy > 0 ? 1.f - fy : 0.f);
  const float az = dz < 0 ? fz : (dz > 0 ? 1.f - fz : 0.f);
  return ax * ax + ay * ay + az * az <= 1.0f + 1e-5f;
}

// Cell lookup over the bounding-box grid of grid_build_device (kernel-level API: loam_b200_tree_build on a map slot).
struct GridCellLookup {
  GridView g;
  GridMeta gm;
  int cx, cy, cz;
  int prune;  // skip the cells of the 3 x 3 x 3 block a query cannot reach (cell_in_reach): pays when the map is beyond L2
  // returns false when no neighbour of the query can hold a point
  __device__ __forceinline__ bool prepare(float qx, float qy, float qz) {
    gm = *g.meta;
    cx = (int)floorf(qx) - gm.ox; cy = (int)floorf(qy) - gm.oy; cz = (int)floorf(qz) - gm.oz;
    return g.m > 0 && !(cx < -1 || cy < -1 || cz < -1 || cx > gm.nx || cy > gm.ny || cz > gm.nz);
  }
  // neighbour cell t = (dz + 1) * 9 + (dy + 1) * 3 + (dx + 1) -> run of its points in `sorted`
  template <bool STATS>
  __device__ __forceinline__ void cell(int t, unsigned& start, unsigned& count, unsigned* stats) const {
    const int z = cz + t / 9 - 1, y = cy + (t / 3) % 3 - 1, x = cx + t % 3 - 1;
    if (z >= 0 && z < gm.nz && y >= 0 && y < gm.ny && x >= 0 && x < gm.nx) {
      const unsigned key = grid_key(gm, x, y, z);
      unsigned h = grid_hash(key) & g.mask;
      uint4 e = __ldg(&g.table[h]);
      if (STATS) stats[0]++;
      while (e.x != 0u && e.x != key + 1u) {
        h = (h + 1) & g.mask;
        e = __ldg(&g.table[h]);
        if (STATS) stats[0]++;
      }
      if (e.x == key + 1u) { start = e.y; count = e.z; }
    }
  }
  __device__ __forceinline__ const float4* points() const { return g.sorted; }
};

// All 8 lanes of the group call this with the same query; on return every lane holds the group's exact 5 nearest
// (d2 < 1.0) in `out` (ascending; id = -1 for missing ones).  gmask = the group's 8 lanes within the warp;
// pre[GRID_SLOTS + 1] / first[GRID_SLOTS] = this group's rows of shared memory.  LOOKUP maps a neighbour cell to its
// run of points (GridCellLookup above, MapCellLookup in mapstore.cuh).
template <bool STATS, typename LOOKUP, int MLP = 2>
__device__ __forceinline__ void grid_knn5_group8(LOOKUP& lk, float qx, float qy, float qz, int sub,
                                                 unsigned gmask, unsigned* pre, unsigned* first, Cand5& out,
                                                 unsigned* stats) {
  Cand5 mine;
#pragma unroll
  for (int i = 0; i < 5; i++) { mine.d[i] = 1.0f; mine.id[i] = -1; }
  const bool inside = lk.prepare(qx, qy, qz);
  const float4* __restrict__ sorted = lk.points();
  if (inside) {  // uniform over the group
    unsigned start[4], count[4];
    const float fx = qx - floorf(qx), fy = qy - floorf(qy), fz = qz - floorf(qz);
#pragma unroll
    for (int r = 0; r < 4; r++) {
      const int t = sub + 8 * r;
      start[r] = 0;
      count[r] = 0;
      if (t < 27 && (!lk.prune || cell_in_reach(t, fx, fy, fz))) lk.template cell<STATS>(t, start[r], count[r], stats);
    }
    // exclusive prefix of the counts in slot order
    const unsigned local = count[0] + count[1] + count[2] + count[3];
    unsigned incl = local;
#pragma unroll
    for (int o = 1; o < 8; o <<= 1) {
      const unsigned y = __shfl_up_sync(gmask, incl, o, 8);
      if (sub >= o) incl += y;
    }
    const unsigned total = __shfl_sync(gmask, incl, 7, 8);
    unsigned run = incl - local;
#pragma unroll
    for (int r = 0; r < 4; r++) {
      pre[sub * 4 + r] = run;
      first[sub * 4 + r] = start[r];
      run += count[r];
    }
    if (sub == 7) pre[GRID_SLOTS] = total;
    __syncwarp(gmask);
    if (STATS && sub == 0) stats[1] += total;
    // lane s takes the CONTIGUOUS range [T s / 8, T (s + 1) / 8) of the flattened list (two loads in flight): its start
    // slot is found by a 5-step binary search, after that the cursor only advances when a cell's run ends.  (A stride-8
    // assignment made every lane walk all 32 slots.)
    const unsigned j_begin = (total * (unsigned)sub) >> 3, j_end = (total * (unsigned)(sub + 1)) >> 3;
    if (j_begin < j_end) {
      unsigned f = 0;
#pragma unroll
      for (int step = 16; step > 0; step >>= 1)
        if (pre[f + step] <= j_begin) f += step;  // last slot whose exclusive prefix is <= j_begin
      unsigned hi = pre[f + 1];
      while (j_begin >= hi) { f++; hi = pre[f + 1]; }  // skip empty slots with the same prefix
      int idx = (int)(first[f] + (j_begin - pre[f]));
      unsigned j = j_begin;
      // MLP loads in flight per lane: the cursor is advanced MLP times first (ALU + shared memory only), then the loads are
      // issued together, then evaluated in order -- the same candidates in the same order for every MLP
      while (j < j_end) {
        int ids[MLP];
#pragma unroll
        for (int u = 0; u < MLP; u++) {
          ids[u] = -1;
          if (j < j_end) {
            ids[u] = idx;
            j++; idx++;
            if (j < j_end && j >= hi) {
              do { f++; hi = pre[f + 1]; } while (j >= hi);
              idx = (int)first[f];
            }
          }
        }
        float4 pp[MLP];
#pragma unroll
        for (int u = 0; u < MLP; u++)
          if (ids[u] >= 0) pp[u] = __ldg(sorted + ids[u]);
#pragma unroll
        for (int u = 0; u < MLP; u++)
          if (ids[u] >= 0) {
            const float dx = qx - pp[u].x, dy = qy - pp[u].y, dz = qz - pp[u].z;
            cand5_offer(mine, dx * dx + dy * dy + dz * dz, ids[u]);
          }
      }
    }
  }
  // merge the eight private lists: five rounds of "smallest head wins, winner advances"
#pragma unroll
  for (int k = 0; k < 5; k++) {
    float bd = mine.d[0];
    int bi = mine.id[0];
#pragma unroll
    for (int o = 4; o > 0; o >>= 1) {
      const float od = __shfl_xor_sync(gmask, bd, o);
      const int oi = __shfl_xor_sync(gmask, bi, o);
      // empty heads (id < 0) never win against a real candidate; among real ones (distance, position) ascending
      const bool take = (oi >= 0) && (bi < 0 || od < bd || (od == bd && oi < bi));
      if (take) { bd = od; bi = oi; }
    }
    out.d[k] = bd;
    out.id[k] = bi;
    if (bi >= 0 && bi == mine.id[0]) {  // my head won: advance
#pragma unroll
      for (int s = 0; s < 4; s++) { mine.d[s] = mine.d[s + 1]; mine.id[s] = mine.id[s + 1]; }
      mine.d[4] = 1.0f;
      mine.id[4] = -1;
    }
  }
}

}  // namespace loamb
