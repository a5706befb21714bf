// Whole-run voxel map (optional, off by default): every registered full-resolution cloud the mapping stage produces is
// accumulated into a device-resident open-addressing hash table of voxels that is never rolled or pruned -- the map of
// the whole run, which the reference itself never keeps (its cube grid forgets cubes that roll out of the window).
//
// Voxel of a point: v_a = (int)floorf(c_a * (1.0f / leaf)) per axis, PCL VoxelGrid's index before it subtracts min_b
// (voxel.cuh: voxel_key_of), so one cloud's voxels form the same partition as VoxelGrid.  Its key is given by the key
// codec below: z-major, so ascending keys are VoxelGrid's output order.  Points that are not finite or whose voxel lies
// outside [-2^20, 2^20) on an axis are skipped (and counted).
//
// One insert of n points:
//   key kernel -> stable two-pass LSD sort of the 64-bit keys (low word, then high word; radix_sort_pairs) -> run heads
//   (voxel_head_kernel + radix_scan_kernel) -> one thread per run: sequential fp64 sums in ascending cloud index, and
//   the run's slot if the voxel is already in the table -> block ranks of the new voxels in key order + scan ->
//   insert (existing voxels add their partial sums, new ones are admitted in ascending key order while the table has
//   room under max_voxels) -> counters.
// Every insert also counts a hit for each voxel that receives points.  The optional visibility pass (before a sweep's
// insert, dense_range_image_kernel + dense_visibility_kernel) counts a miss for every stored voxel that the sweep sees
// through: its pixel of the sweep's range image holds a return farther than the centroid's range + margin.  Its other
// mode, carve mode (dense_carve_mark_kernel + dense_carve_kernel), walks every point's ray through a live occupancy
// index of the table instead and counts one miss for every stored voxel a ray crosses short of its return.
// Per voxel the table keeps count and the fp64 sums S = ((P1 + P2) + P3) + ... of the per-sweep partial sums; export
// gives (float)(S / count) per field in ascending key order, so the result does not depend on where the hash placed
// an entry.  Keys are unique within one insert, so no value update needs an atomic.
#pragma once

#include <cmath>
#include <vector>

#include "linalg.cuh"
#include "mapping_lm.cuh"
#include "voxel.cuh"

namespace loamb {

constexpr unsigned long long DENSE_EMPTY = ~0ull;  // empty table slot; also the key of a skipped point (sorts last)

// ---- voxel key codec: the only statement of the key layout.  Voxel (v_x, v_y, v_z) has the biased indices
// u_a = v_a + 2^20 in [0, 2^21) and the key u_z << 42 | u_y << 21 | u_x.  Its 8^3 brick has the key
// (u_z >> 3) << 36 | (u_y >> 3) << 18 | (u_x >> 3), and its bit in the brick's 512-bit mask is
// (u_z & 7) << 6 | (u_y & 7) << 3 | (u_x & 7).
constexpr int DENSE_KEY_BIAS = 1 << 20;                 // voxels per half axis
constexpr int DENSE_AXIS = 2 * DENSE_KEY_BIAS;          // biased indices per axis
constexpr unsigned long long DENSE_AXIS_MASK = DENSE_AXIS - 1;
constexpr float DENSE_KEY_LIM = (float)DENSE_KEY_BIAS;

__device__ __forceinline__ unsigned long long dense_pack(unsigned ux, unsigned uy, unsigned uz) {
  return ((unsigned long long)uz << 42) | ((unsigned long long)uy << 21) | (unsigned long long)ux;
}

// key of voxel (vx, vy, vz), each inside [-2^20, 2^20)
__device__ __forceinline__ unsigned long long dense_key(int vx, int vy, int vz) {
  return dense_pack((unsigned)(vx + DENSE_KEY_BIAS), (unsigned)(vy + DENSE_KEY_BIAS), (unsigned)(vz + DENSE_KEY_BIAS));
}

__device__ __forceinline__ void dense_unpack(unsigned long long key, int& ux, int& uy, int& uz) {
  ux = (int)(key & DENSE_AXIS_MASK);
  uy = (int)((key >> 21) & DENSE_AXIS_MASK);
  uz = (int)(key >> 42);
}

__device__ __forceinline__ unsigned long long dense_brick(int ux, int uy, int uz) {
  return ((unsigned long long)(uz >> 3) << 36) | ((unsigned long long)(uy >> 3) << 18) | (unsigned long long)(ux >> 3);
}

__device__ __forceinline__ unsigned dense_brick_bit(int ux, int uy, int uz) {
  return ((unsigned)(uz & 7) << 6) | ((unsigned)(uy & 7) << 3) | (unsigned)(ux & 7);
}

// host: the voxel floor(o / leaf) of coordinate o lies inside the key range (NaN and +-inf do not)
inline bool dense_in_key_range(double o, double leaf) {
  const double v = std::floor(o / leaf);
  return v >= -(double)DENSE_KEY_BIAS && v < (double)DENSE_KEY_BIAS;
}

struct __align__(16) DenseSlot {  // 48 B
  unsigned long long key;
  unsigned count;
  unsigned evidence;              // hits (low 16 bits) and misses (high 16 bits), each saturating at 65535
  double sum[4];                  // x, y, z, intensity
};

constexpr unsigned DENSE_EVIDENCE_NEW = 1u;  // a voxel's first insert: 1 hit, 0 misses

__device__ __forceinline__ unsigned dense_add_hit(unsigned e) { return (e & 0xffffu) == 0xffffu ? e : e + 1u; }
__device__ __forceinline__ unsigned dense_add_miss(unsigned e) { return (e >> 16) == 0xffffu ? e : e + 0x10000u; }

struct DenseCounters {
  unsigned long long voxels, skipped, dropped;
  unsigned long long bricks;  // bricks of carve mode's occupancy index (0 while carve mode is off)
};

// per-run results of one insert (indexed by run = voxel rank in key order)
struct DenseRuns {
  unsigned long long* key;
  unsigned* count;
  double4* sum;
  long long* slot;  // table slot of a voxel already in the map, -1 new, -2 the run of skipped points
};

__device__ __forceinline__ unsigned long long dense_key_of(const float4& q, float inv) {
  const float fx = floorf(q.x * inv), fy = floorf(q.y * inv), fz = floorf(q.z * inv);
  // NaN fails every comparison; +-inf and out-of-range voxels fail the bounds (compared before the int conversion)
  if (!(fx >= -DENSE_KEY_LIM && fx < DENSE_KEY_LIM && fy >= -DENSE_KEY_LIM && fy < DENSE_KEY_LIM &&
        fz >= -DENSE_KEY_LIM && fz < DENSE_KEY_LIM))
    return DENSE_EMPTY;
  return dense_key((int)fx, (int)fy, (int)fz);
}

// 64-bit finaliser of splitmix64: consecutive voxel keys spread over the whole table
__device__ __forceinline__ unsigned long long dense_hash(unsigned long long k) {
  k ^= k >> 30;
  k *= 0xbf58476d1ce4e5b9ull;
  k ^= k >> 27;
  k *= 0x94d049bb133111ebull;
  k ^= k >> 31;
  return k;
}

__device__ __forceinline__ long long dense_find(const DenseSlot* __restrict__ t, unsigned long long mask,
                                                unsigned long long key) {
  unsigned long long h = dense_hash(key) & mask;
  for (;;) {
    const unsigned long long k = t[h].key;
    if (k == key) return (long long)h;
    if (k == DENSE_EMPTY) return -1;
    h = (h + 1) & mask;
  }
}

// claim an empty slot for `key` (absent from the table; load factor <= 0.5, so the probe ends)
__device__ __forceinline__ unsigned long long dense_claim(DenseSlot* t, unsigned long long mask, unsigned long long key) {
  unsigned long long h = dense_hash(key) & mask;
  while (atomicCAS(&t[h].key, DENSE_EMPTY, key) != DENSE_EMPTY) h = (h + 1) & mask;
  return h;
}

// 64-bit key per point + the (low word, index) pairs of the first sort pass
__global__ void dense_key_kernel(const float4* __restrict__ p, int n, float inv, unsigned long long* __restrict__ keys64,
                                 unsigned* __restrict__ keys_lo, int* __restrict__ vals) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const unsigned long long k = dense_key_of(p[i], inv);
  keys64[i] = k;
  keys_lo[i] = (unsigned)k;
  vals[i] = i;
}

// export: the (low word, index) pairs of the compacted keys
__global__ void dense_lo_kernel(const unsigned long long* __restrict__ keys64, int n, unsigned* __restrict__ keys_lo,
                                int* __restrict__ vals) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  keys_lo[i] = (unsigned)keys64[i];
  vals[i] = i;
}

// second pass input: high words in the order of the first pass (stable passes keep the index order inside a key)
__global__ void dense_hi_kernel(const unsigned long long* __restrict__ keys64, const int* order, int n,
                                unsigned* keys_hi, int* vals) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int o = order[i];  // order may alias vals: read before the write
  keys_hi[i] = (unsigned)(keys64[o] >> 32);
  vals[i] = o;
}

__global__ void dense_gather_keys_kernel(const unsigned long long* __restrict__ keys64, const int* __restrict__ order,
                                         int n, unsigned long long* __restrict__ sorted) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) sorted[i] = keys64[order[i]];
}

// one thread per run head (sorted position i): the run's points in ascending cloud index, each float converted to
// double and added in that order; then the voxel's slot if the table already holds it
__global__ void dense_run_kernel(const float4* __restrict__ p, const unsigned long long* __restrict__ skey,
                                 const int* __restrict__ order, const unsigned* __restrict__ pos,
                                 const unsigned* __restrict__ block_off, int n, const DenseSlot* __restrict__ table,
                                 unsigned long long mask, DenseRuns runs, DenseCounters* __restrict__ ctr) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const unsigned pv = pos[i];
  if (!(pv >> 31)) return;
  const unsigned r = (pv & 0x7fffffffu) + block_off[i / SCAN_BS];
  const unsigned long long k = skey[i];
  double sx = 0.0, sy = 0.0, sz = 0.0, si = 0.0;
  unsigned cnt = 0;
  for (int u = i; u < n && skey[u] == k; u++) {
    const float4 q = p[order[u]];
    sx += (double)q.x;
    sy += (double)q.y;
    sz += (double)q.z;
    si += (double)q.w;
    cnt++;
  }
  runs.key[r] = k;
  runs.count[r] = cnt;
  if (k == DENSE_EMPTY) {  // the skipped points: one run, the last
    runs.slot[r] = -2;
    ctr->skipped += cnt;
    return;
  }
  runs.sum[r] = make_double4(sx, sy, sz, si);
  runs.slot[r] = dense_find(table, mask, k);
}

// exclusive rank of every new voxel among the new voxels of its block (runs are in key order) + per-block totals
__global__ void __launch_bounds__(SCAN_BS)
dense_new_rank_kernel(const long long* __restrict__ slot, const int* __restrict__ n_runs, int bound,
                      unsigned* __restrict__ rank, unsigned* __restrict__ block_sums) {
  __shared__ unsigned ws[32];
  const int r = blockIdx.x * SCAN_BS + threadIdx.x;
  const int m = min(bound, *n_runs);
  const unsigned f = (r < m && slot[r] == -1) ? 1u : 0u;
  unsigned x = f;
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
  if (r < bound) rank[r] = incl - f;
  if (threadIdx.x == SCAN_BS - 1) block_sums[blockIdx.x] = incl;
}

// existing voxels add the run's partial sums; a new voxel is admitted when fewer than max_voxels - voxels new voxels
// precede it in key order, otherwise its points are dropped.  ctr->voxels is read here and advanced by
// dense_finish_kernel afterwards.
__global__ void dense_insert_kernel(DenseRuns runs, const int* __restrict__ n_runs, const unsigned* __restrict__ rank,
                                    const unsigned* __restrict__ block_off, DenseSlot* table, unsigned long long mask,
                                    DenseCounters* __restrict__ ctr, unsigned long long max_voxels) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= *n_runs) return;
  const long long s = runs.slot[r];
  if (s == -2) return;
  const double4 p = runs.sum[r];
  const unsigned cnt = runs.count[r];
  if (s >= 0) {
    DenseSlot& e = table[s];
    e.count += cnt;
    e.evidence = dense_add_hit(e.evidence);
    e.sum[0] += p.x;
    e.sum[1] += p.y;
    e.sum[2] += p.z;
    e.sum[3] += p.w;
    return;
  }
  const unsigned long long nr = rank[r] + block_off[r / SCAN_BS];
  if (ctr->voxels + nr >= max_voxels) {
    atomicAdd(&ctr->dropped, (unsigned long long)cnt);
    return;
  }
  DenseSlot& e = table[dense_claim(table, mask, runs.key[r])];
  e.count = cnt;
  e.evidence = DENSE_EVIDENCE_NEW;
  e.sum[0] = p.x;
  e.sum[1] = p.y;
  e.sum[2] = p.z;
  e.sum[3] = p.w;
}

__global__ void dense_finish_kernel(DenseCounters* ctr, const int* __restrict__ new_total, unsigned long long max_voxels) {
  if (threadIdx.x != 0) return;
  // the cap may have been lowered below the stored voxels (loam_b200_dense_enable): then no room at all
  const unsigned long long room = ctr->voxels < max_voxels ? max_voxels - ctr->voxels : 0ull;
  const unsigned long long nt = (unsigned long long)*new_total;
  ctr->voxels += nt < room ? nt : room;
}

// growth: every entry of the old table moves to the new one (each key once, so a plain claim suffices)
__global__ void dense_rehash_kernel(const DenseSlot* __restrict__ old_t, unsigned long long old_size, DenseSlot* t,
                                   unsigned long long mask) {
  const unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x;
  if (i >= old_size) return;
  const DenseSlot e = old_t[i];
  if (e.key == DENSE_EMPTY) return;
  t[dense_claim(t, mask, e.key)] = e;
}

// export: occupied slots -> counter[0]; those with (double)misses <= max_miss_ratio * (double)hits -> (key, slot) in any
// order (sorted by key afterwards) and counter[1]; at most cap are written (the caller checks counter[0] against the
// voxel counter).  max_miss_ratio = +inf keeps every voxel (hits >= 1 for every stored one).
__global__ void dense_compact_kernel(const DenseSlot* __restrict__ t, unsigned long long size,
                                     unsigned long long* __restrict__ keys, int* __restrict__ slots,
                                     unsigned* __restrict__ counter, unsigned cap, double max_miss_ratio) {
  const unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x;
  if (i >= size) return;
  const unsigned long long k = t[i].key;
  if (k == DENSE_EMPTY) return;
  atomicAdd(&counter[0], 1u);
  const unsigned ev = t[i].evidence;
  if (!((double)(ev >> 16) <= max_miss_ratio * (double)(ev & 0xffffu))) return;
  const unsigned d = atomicAdd(&counter[1], 1u);
  if (d >= cap) return;
  keys[d] = k;
  slots[d] = (int)i;
}

__global__ void dense_centroid_kernel(const DenseSlot* __restrict__ t, const int* __restrict__ slots,
                                      const int* __restrict__ order, int m, float4* __restrict__ out,
                                      unsigned* __restrict__ counts, unsigned* __restrict__ evidence) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= m) return;
  const DenseSlot& e = t[slots[order[i]]];
  const double c = (double)e.count;
  out[i] = make_float4((float)(e.sum[0] / c), (float)(e.sum[1] / c), (float)(e.sum[2] / c), (float)(e.sum[3] / c));
  if (counts) counts[i] = e.count;
  if (evidence) evidence[i] = e.evidence;
}

// ---- snapshots and merging (include/loam_b200.h "Whole-run voxel map snapshots and merging")
// snapshot: the raw slot fields of the m compacted voxels in the sort's (ascending key) order
__global__ void dense_snapshot_kernel(const DenseSlot* __restrict__ t, const int* __restrict__ slots,
                                      const int* __restrict__ order, int m, unsigned long long* __restrict__ keys,
                                      unsigned* __restrict__ counts, unsigned* __restrict__ evidence,
                                      double4* __restrict__ sums) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= m) return;
  const DenseSlot& e = t[slots[order[i]]];
  keys[i] = e.key;
  counts[i] = e.count;
  evidence[i] = e.evidence;
  sums[i] = make_double4(e.sum[0], e.sum[1], e.sum[2], e.sum[3]);
}

// rotation and translation of a merge, by value in the kernel arguments (on == 0: the sums are taken as they are)
struct DenseMergePose {
  double cx, sx, cy, sy, cz, sz;  // std::cos / std::sin of the pose's float rot_x, rot_y, rot_z (host)
  double px, py, pz;              // the pose's float pos
  int on;
};

// merge, one thread per entry, fp64 without FMA: S' = rotZ, rotX, rotY of (Sx, Sy, Sz) (dense_raycast's order) +
// count * pos per axis, intensity unchanged (in place); the destination key is that of the fp32 centroid
// (float)(S' / count) by the map's rule, DENSE_EMPTY when it is not finite or outside the key range.  Also the
// (low word, index) pairs of the first sort pass.
__global__ void dense_merge_key_kernel(double4* __restrict__ sums, const unsigned* __restrict__ counts, int n,
                                       DenseMergePose a, float inv, unsigned long long* __restrict__ keys64,
                                       unsigned* __restrict__ keys_lo, int* __restrict__ vals) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  double4 s = sums[i];
  const double c = (double)counts[i];
  if (a.on) {
    const double x1 = a.cz * s.x - a.sz * s.y, y1 = a.sz * s.x + a.cz * s.y;
    const double y2 = a.cx * y1 - a.sx * s.z, z2 = a.sx * y1 + a.cx * s.z;
    s.x = (a.cy * x1 + a.sy * z2) + c * a.px;
    s.y = y2 + c * a.py;
    s.z = (a.cy * z2 - a.sy * x1) + c * a.pz;
    sums[i] = s;
  }
  const unsigned long long k =
      dense_key_of(make_float4((float)(s.x / c), (float)(s.y / c), (float)(s.z / c), 0.f), inv);
  keys64[i] = k;
  keys_lo[i] = (unsigned)k;
  vals[i] = i;
}

__device__ __forceinline__ unsigned dense_add_evidence(unsigned a, unsigned b) {
  const unsigned h = (a & 0xffffu) + (b & 0xffffu), m = (a >> 16) + (b >> 16);
  return (h < 0xffffu ? h : 0xffffu) | ((m < 0xffffu ? m : 0xffffu) << 16);
}

// merge, one thread per run head (sorted position i) -- dense_run_kernel over entries: the group's sums
// ((0.0 + S'_1) + S'_2) + ... in ascending input index, counts added in uint32, hits and misses each added with
// saturation; then the voxel's slot if the table already holds it.  The skipped entries (key DENSE_EMPTY, the last run)
// add their counts to ctr->skipped.
__global__ void dense_merge_run_kernel(const double4* __restrict__ sums, const unsigned* __restrict__ counts,
                                       const unsigned* __restrict__ evidence, const unsigned long long* __restrict__ skey,
                                       const int* __restrict__ order, const unsigned* __restrict__ pos,
                                       const unsigned* __restrict__ block_off, int n, const DenseSlot* __restrict__ table,
                                       unsigned long long mask, DenseRuns runs, unsigned* __restrict__ run_ev,
                                       DenseCounters* __restrict__ ctr) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const unsigned pv = pos[i];
  if (!(pv >> 31)) return;
  const unsigned r = (pv & 0x7fffffffu) + block_off[i / SCAN_BS];
  const unsigned long long k = skey[i];
  double sx = 0.0, sy = 0.0, sz = 0.0, si = 0.0;
  unsigned long long cnt = 0;
  unsigned ev = 0;
  for (int u = i; u < n && skey[u] == k; u++) {
    const int o = order[u];
    const double4 s = sums[o];
    sx += s.x;
    sy += s.y;
    sz += s.z;
    si += s.w;
    cnt += counts[o];
    ev = dense_add_evidence(ev, evidence[o]);
  }
  runs.key[r] = k;
  runs.count[r] = (unsigned)cnt;
  if (k == DENSE_EMPTY) {
    runs.slot[r] = -2;
    ctr->skipped += cnt;
    return;
  }
  runs.sum[r] = make_double4(sx, sy, sz, si);
  run_ev[r] = ev;
  runs.slot[r] = dense_find(table, mask, k);
}

// merge -- dense_insert_kernel with the evidence of the runs instead of one hit per insert
__global__ void dense_merge_insert_kernel(DenseRuns runs, const unsigned* __restrict__ run_ev,
                                          const int* __restrict__ n_runs, const unsigned* __restrict__ rank,
                                          const unsigned* __restrict__ block_off, DenseSlot* table,
                                          unsigned long long mask, DenseCounters* __restrict__ ctr,
                                          unsigned long long max_voxels) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= *n_runs) return;
  const long long s = runs.slot[r];
  if (s == -2) return;
  const double4 p = runs.sum[r];
  const unsigned cnt = runs.count[r];
  if (s >= 0) {
    DenseSlot& e = table[s];
    e.count += cnt;
    e.evidence = dense_add_evidence(e.evidence, run_ev[r]);
    e.sum[0] += p.x;
    e.sum[1] += p.y;
    e.sum[2] += p.z;
    e.sum[3] += p.w;
    return;
  }
  const unsigned long long nr = rank[r] + block_off[r / SCAN_BS];
  if (ctr->voxels + nr >= max_voxels) {
    atomicAdd(&ctr->dropped, (unsigned long long)cnt);
    return;
  }
  DenseSlot& e = table[dense_claim(table, mask, runs.key[r])];
  e.count = cnt;
  e.evidence = run_ev[r];
  e.sum[0] = p.x;
  e.sum[1] = p.y;
  e.sum[2] = p.z;
  e.sum[3] = p.w;
}

// ---- normals of the exported cloud (include/loam_b200.h "loam_b200_dense_export_normals")
// first position in [lo, hi) of the ascending keys whose key is >= `key`
__device__ __forceinline__ int dense_lower_bound(const unsigned long long* __restrict__ k, int lo, int hi,
                                                 unsigned long long key) {
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (k[mid] < key) lo = mid + 1;
    else hi = mid;
  }
  return lo;
}

// Calls visit(j) for every position j in [0, n) of the ascending keys skey whose voxel lies within `radius` voxels of
// `key`'s on every axis, in ascending key order: per (z, y) row inside the key range, a lower bound of the row's first
// key (x clamped to the range), then forward while the key stays in the row.  Rows outside the range are skipped, so an
// offset never wraps into the next row or plane.  The order is load-bearing: it fixes the fp64 sums of the normals and
// the first-smallest tie rule of the alignment's match.
template <typename F>
__device__ __forceinline__ void dense_box_walk(const unsigned long long* __restrict__ skey, int n, unsigned long long key,
                                               int radius, F&& visit) {
  int vx, vy, vz;
  dense_unpack(key, vx, vy, vz);
  const unsigned long long x0 = (unsigned long long)max(vx - radius, 0);
  const unsigned long long x1 = (unsigned long long)min(vx + radius, DENSE_AXIS - 1);
  int lo = 0;  // rows ascend in key order: each row's search starts where the previous row ended
  for (int z = vz - radius; z <= vz + radius; z++) {
    if (z < 0 || z >= DENSE_AXIS) continue;
    for (int y = vy - radius; y <= vy + radius; y++) {
      if (y < 0 || y >= DENSE_AXIS) continue;
      const unsigned long long row = dense_pack(0u, (unsigned)y, (unsigned)z);
      const unsigned long long last = row | x1;
      int j = dense_lower_bound(skey, lo, n, row | x0);
      for (; j < n && skey[j] <= last; j++) visit(j);
      lo = j;
    }
  }
}

// One thread per exported voxel, over the export's own arrays (keys ascending, centroids in the same order), so the
// miss-ratio filter is already applied and the table is never touched.  Neighbours: the exported voxels of
// dense_box_walk.  Centred fp64 sums of the fp32 centroids, covariance rounded to fp32 once per entry, sym_eigen<3>,
// curvature ev0 / (ev0 + ev1 + ev2), normal flipped towards the viewpoint.  Fewer than 3 neighbours, or no
// convergence: NaN normal and curvature.  The library is built without FMA contraction, so every product and sum
// rounds on its own, as in tests/normals_reference.py.
__global__ void __launch_bounds__(128)
dense_normals_kernel(const unsigned long long* __restrict__ skey, const float4* __restrict__ cent, int n, int radius,
                     double3 vp, float4* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const unsigned long long key = skey[i];
  const float4 cv = cent[i];
  const double cx = (double)cv.x, cy = (double)cv.y, cz = (double)cv.z;
  double s1x = 0.0, s1y = 0.0, s1z = 0.0, sxx = 0.0, sxy = 0.0, sxz = 0.0, syy = 0.0, syz = 0.0, szz = 0.0;
  int k = 0;
  dense_box_walk(skey, n, key, radius, [&](int j) {
    const float4 cw = cent[j];
    const double dx = (double)cw.x - cx, dy = (double)cw.y - cy, dz = (double)cw.z - cz;
    s1x += dx;
    s1y += dy;
    s1z += dz;
    sxx += dx * dx;
    sxy += dx * dy;
    sxz += dx * dz;
    syy += dy * dy;
    syz += dy * dz;
    szz += dz * dz;
    k++;
  });
  const float qnan = __int_as_float(0x7fc00000);
  if (k < 3) {
    out[i] = make_float4(qnan, qnan, qnan, qnan);
    return;
  }
  const double kd = (double)k;
  float m[9];
  m[0] = (float)((sxx - (s1x * s1x) / kd) / kd);  // (0,0)
  m[1] = (float)((sxy - (s1x * s1y) / kd) / kd);  // (1,0)
  m[2] = (float)((sxz - (s1x * s1z) / kd) / kd);  // (2,0)
  m[4] = (float)((syy - (s1y * s1y) / kd) / kd);  // (1,1)
  m[5] = (float)((syz - (s1y * s1z) / kd) / kd);  // (2,1)
  m[8] = (float)((szz - (s1z * s1z) / kd) / kd);  // (2,2)
  m[3] = m[6] = m[7] = 0.f;                       // upper triangle: never read
  float ev[3], V[9];
  if (!sym_eigen<3>(m, ev, V)) {
    out[i] = make_float4(qnan, qnan, qnan, qnan);
    return;
  }
  float nx = V[0], ny = V[1], nz = V[2];
  const float den = (ev[0] + ev[1]) + ev[2];
  const float curv = den == 0.f ? 0.f : ev[0] / den;
  if (((vp.x - cx) * (double)nx + (vp.y - cy) * (double)ny) + (vp.z - cz) * (double)nz < 0.0) {
    nx = -nx;
    ny = -ny;
    nz = -nz;
  }
  out[i] = make_float4(nx, ny, nz, curv);
}

// ---- registration target (include/loam_b200.h "loam_b200_dense_target_build" / "_load" / "_align_iterate")
// load: one thread per sorted entry -- gather key, centroid and normal in key order; flag a key outside the range
// (DENSE_EMPTY sorts last) with bit 0 and a key equal to its predecessor's with bit 1
__global__ void dense_target_gather_kernel(const unsigned long long* __restrict__ keys64, const int* __restrict__ order,
                                           int n, const float4* __restrict__ cent_in, const float4* __restrict__ nrm_in,
                                           unsigned long long* __restrict__ skey, float4* __restrict__ cent,
                                           float4* __restrict__ nrm, int* __restrict__ bad) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int o = order[i];
  const unsigned long long k = keys64[o];
  skey[i] = k;
  cent[i] = cent_in[o];
  nrm[i] = nrm_in[o];
  if (k == DENSE_EMPTY) atomicOr(bad, 1);
  else if (i > 0 && keys64[order[i - 1]] == k) atomicOr(bad, 2);
}

// The alignment's match of a map-frame point q whose voxel is `key`: among the target voxels of dense_box_walk that
// use(j) admits, the first smallest d2 = (dx*dx + dy*dy) + dz*dz, d = c - q in fp32, below the gate (strict <); -1
// when none.  dense_align_kernel admits the voxels with a normal, dense_ground_cloud_kernel the ground voxels.
template <typename F>
__device__ __forceinline__ int dense_match(const unsigned long long* __restrict__ skey, const float4* __restrict__ cent,
                                           int m, unsigned long long key, int radius, float gate, float qx, float qy,
                                           float qz, F&& use) {
  int best = -1;
  float best_d2 = gate;  // strict < from the gate: the first smallest d2 below it
  dense_box_walk(skey, m, key, radius, [&](int j) {
    if (!use(j)) return;
    const float4 c = cent[j];
    const float dx = c.x - qx, dy = c.y - qy, dz = c.z - qz;
    const float d2 = (dx * dx + dy * dy) + dz * dz;
    if (d2 < best_d2) {
      best_d2 = d2;
      best = j;
    }
  });
  return best;
}

// One Gauss-Newton iteration of a cloud against the target, one thread per point (point i in CTA i / LM_THREADS):
//   q = associate_to_map(pose, p); v = voxel of q (dense_key_of with the target's leaf);
//   candidates: the target voxels of dense_box_walk around v whose normal_x is not NaN; the first smallest d2 = (dx*dx + dy*dy) + dz*dz, d = c - q, wins when d2 < gate;
//   pd2 = (nx*(qx - cx) + ny*(qy - cy)) + nz*(qz - cz); s = 1 - 0.9f*|pd2| / sqrtf(sqrtf(|p|^2)) with the SENSOR-frame p;
//   selected when (double)s > 0.1; coeff = s * (n, pd2); Jacobian row and rhs of the scan-to-map kernels.
// Slots 0..26 of the 32 sums: AtA (upper triangle) and AtB; 27: selected rows; 28: sum of pd2^2 over them.  The
// reduction is reduce_normal_equations (fp32 xor butterfly per warp, the 4 warp sums in warp order, CTA partials folded
// in double in fixed order).  The library is built without FMA contraction, as tests/align_reference.py assumes.
//
// Hypotheses (loam_b200_dense_score / _align_batch): blockIdx.y is the entry of the launch's hypothesis list; entry h
// reads its pose from args[h] and owns partials [h][gridDim.x][stride], result [h][stride] and ticket [h], so one
// launch evaluates one cloud at every pose of the list and each entry's sums are those of a launch at that pose alone.
// A single pose is the list of one; the full kernel then takes it by value (LIST = false: the pose `one`, no copy
// before the launch, read from the parameter bank).  SCORE: only slots 27 and 28 are summed (stride DENSE_SCORE_NEQ), each in the
// order reduce_normal_equations sums it, so their bits are the full kernel's; the Jacobian row is not formed.
constexpr int DENSE_SCORE_NEQ = 2;  // the score's slots: selected rows, sum of pd2^2

// reduce_normal_equations restricted to the two score slots (partials and result of stride DENSE_SCORE_NEQ): per slot
// the same fp32 butterfly, warp order and double fold over the CTA partials, so each slot's bits are that function's
__device__ __forceinline__ void reduce_score_sums(float n_sel, float sum_sq, float* __restrict__ partials,
                                                  float* __restrict__ result, unsigned int* ticket, unsigned n_blocks) {
  __shared__ float s_part[LM_THREADS / 32][DENSE_SCORE_NEQ];
  __shared__ bool s_last;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float v0 = n_sel, v1 = sum_sq;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    v0 += __shfl_xor_sync(0xffffffffu, v0, o);
    v1 += __shfl_xor_sync(0xffffffffu, v1, o);
  }
  if (lane == 0) {
    s_part[warp][0] = v0;
    s_part[warp][1] = v1;
  }
  __syncthreads();
  if (threadIdx.x < DENSE_SCORE_NEQ) {
    float v = 0.f;
    for (int wv = 0; wv < LM_THREADS / 32; wv++) v += s_part[wv][threadIdx.x];
    __stcg(&partials[(size_t)blockIdx.x * DENSE_SCORE_NEQ + threadIdx.x], v);
  }
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) s_last = (atomicAdd(ticket, 1u) == n_blocks - 1);
  __syncthreads();
  if (s_last) {
    __threadfence();
    __shared__ double s_fold[LM_THREADS / 32][DENSE_SCORE_NEQ];
    if (lane < DENSE_SCORE_NEQ) {
      double v = 0.0;
      for (unsigned bk = warp; bk < n_blocks; bk += LM_THREADS / 32)
        v += (double)__ldcg(&partials[(size_t)bk * DENSE_SCORE_NEQ + lane]);
      s_fold[warp][lane] = v;
    }
    __syncthreads();
    if (threadIdx.x < DENSE_SCORE_NEQ) {
      double v = 0.0;
      for (int wv = 0; wv < LM_THREADS / 32; wv++) v += s_fold[wv][threadIdx.x];
      result[threadIdx.x] = (float)v;
    }
    if (threadIdx.x == 0) *ticket = 0u;
  }
}

template <bool SCORE, bool LIST>
__global__ void __launch_bounds__(LM_THREADS)
dense_align_kernel(const unsigned long long* __restrict__ skey, const float4* __restrict__ cent,
                   const float4* __restrict__ nrm, int m, float inv, int radius, float gate,
                   const float4* __restrict__ pts, int n, MapIterArgs one, const MapIterArgs* __restrict__ args,
                   float* __restrict__ partials, float* __restrict__ result, unsigned int* ticket,
                   int* __restrict__ dbg_match, float4* __restrict__ dbg_coeff, int8_t* __restrict__ dbg_sel) {
  constexpr int NACC = SCORE ? DENSE_SCORE_NEQ : 29;
  constexpr int SLOT_SEL = SCORE ? 0 : 27, SLOT_SQ = SCORE ? 1 : 28;
  constexpr int WORDS = (int)(sizeof(MapIterArgs) / sizeof(float));
  static_assert(WORDS <= LM_THREADS, "one thread per word of the pose");
  static_assert(LIST || !SCORE, "the score always reads a pose list");
  __shared__ MapIterArgs s_args;  // LIST: this entry's pose, read from shared memory by every thread
  if constexpr (LIST) {
    if (threadIdx.x < WORDS)
      reinterpret_cast<float*>(&s_args)[threadIdx.x] = reinterpret_cast<const float*>(args + blockIdx.y)[threadIdx.x];
    __syncthreads();
  }
  const MapIterArgs& a = LIST ? s_args : one;  // !LIST: the single pose, a kernel parameter as before the list
  const int stride = SCORE ? DENSE_SCORE_NEQ : NEQ;
  partials += (size_t)blockIdx.y * gridDim.x * stride;
  result += (size_t)blockIdx.y * stride;
  ticket += blockIdx.y;
  float acc[NACC];
#pragma unroll
  for (int k = 0; k < NACC; k++) acc[k] = 0.f;
  const int i = blockIdx.x * LM_THREADS + threadIdx.x;
  if (i < n) {  // every thread takes part in the reduction below
    const float4 po = pts[i];
    int best = -1;
    float4 coeff = make_float4(0.f, 0.f, 0.f, 0.f);
    bool sel = false;
    if (isfinite(po.x) && isfinite(po.y) && isfinite(po.z)) {
      float qx, qy, qz;
      associate_to_map(a, po, qx, qy, qz);
      const unsigned long long key = dense_key_of(make_float4(qx, qy, qz, 0.f), inv);
      if (key != DENSE_EMPTY)
        best = dense_match(skey, cent, m, key, radius, gate, qx, qy, qz, [&](int j) { return !isnan(nrm[j].x); });
      if (best >= 0) {
        const float4 c = cent[best], nv = nrm[best];
        const float pd2 = (nv.x * (qx - c.x) + nv.y * (qy - c.y)) + nv.z * (qz - c.z);
        const float s = 1.f - 0.9f * fabsf(pd2) / sqrtf(sqrtf(po.x * po.x + po.y * po.y + po.z * po.z));
        coeff = make_float4(s * nv.x, s * nv.y, s * nv.z, s * pd2);
        sel = (double)s > 0.1;
        if (sel) {
          if constexpr (!SCORE) {
            float row[6], rhs;
            map_jacobian_row(a, po, coeff, row, rhs);
            int k = 0;
#pragma unroll
            for (int r = 0; r < 6; r++)
#pragma unroll
              for (int t = r; t < 6; t++) acc[k++] = row[r] * row[t];
#pragma unroll
            for (int r = 0; r < 6; r++) acc[21 + r] = row[r] * rhs;
          }
          acc[SLOT_SEL] = 1.f;
          acc[SLOT_SQ] = pd2 * pd2;
        }
      }
    }
    if (!SCORE && dbg_match) {  // a single pose only
      dbg_match[i] = best;
      dbg_coeff[i] = coeff;
      dbg_sel[i] = sel ? 1 : 0;
    }
  }
  if constexpr (SCORE)
    reduce_score_sums(acc[0], acc[1], partials, result, ticket, gridDim.x);
  else
    reduce_normal_equations(acc, partials, result, ticket, ResultMailbox{nullptr, 0}, gridDim.x);
}

// ---- visibility pass: one sweep's sensor pose and range image (include/loam_b200.h "loam_b200_dense_visibility")
constexpr double DENSE_RAD2DEG = 180.0 / 3.14159265358979323846;
constexpr unsigned DENSE_NO_RETURN = 0xffffffffu;  // empty pixel (above the bits of +inf, like every float bit pattern
                                                   // of a non-negative float is below it)

struct DenseView {                // by value in the kernel arguments
  double px, py, pz;              // sensor position (the pose's float pos)
  double cy, sy, cx, sx, cz, sz;  // cos / sin of -rot_y, -rot_x, -rot_z (double, computed by the host)
  double h_res, v_res, margin;    // degrees, degrees, metres
  int rows, cols;
};

// map-frame position -> range and pixel in the sensor frame of `v`, all in double: pointAssociateTobeMapped
// (BasicLaserMapping.cpp:223-231: the offset, then rotY, rotX, rotZ of math_utils.h); elevation atan2(y, |(x, z)|)
// (y up), azimuth atan2(x, z).  The library is built without FMA contraction, so every product and sum rounds on its
// own, as in tests/visibility_reference.py.
__device__ __forceinline__ int dense_pixel(const DenseView& v, double x, double y, double z, double& r) {
  x -= v.px;
  y -= v.py;
  z -= v.pz;
  double t = x;  // rotY
  x = v.cy * t + v.sy * z;
  z = v.cy * z - v.sy * t;
  t = y;  // rotX
  y = v.cx * t - v.sx * z;
  z = v.sx * t + v.cx * z;
  t = x;  // rotZ
  x = v.cz * t - v.sz * y;
  y = v.sz * t + v.cz * y;
  r = sqrt((x * x + y * y) + z * z);
  const double e = atan2(y, sqrt(x * x + z * z));
  const double a = atan2(x, z);
  const double fr = floor((e * DENSE_RAD2DEG + 90.0) / v.v_res);
  const double fc = floor((a * DENSE_RAD2DEG + 180.0) / v.h_res);
  const int row = fr < 0.0 ? 0 : (fr > (double)(v.rows - 1) ? v.rows - 1 : (int)fr);
  int col = (int)((long long)fc % v.cols);
  if (col < 0) col += v.cols;
  return row * v.cols + col;
}

// one thread per point: the minimum range per pixel over the finite points with r > 0 (float bits of non-negative
// floats order like the floats, so atomicMin gives the same image in any order)
__global__ void dense_range_image_kernel(const float4* __restrict__ p, int n, DenseView v, unsigned* __restrict__ img) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float4 q = p[i];
  if (!(isfinite(q.x) && isfinite(q.y) && isfinite(q.z))) return;
  double r;
  const int pix = dense_pixel(v, (double)q.x, (double)q.y, (double)q.z, r);
  if (r > 0.0) atomicMin(&img[pix], __float_as_uint((float)r));
}

// one thread per table slot (grid-stride): a stored voxel whose pixel holds a finite return farther than its
// centroid's range + margin is seen through -> one more miss.  Pixels without a return are no evidence.
__global__ void dense_visibility_kernel(DenseSlot* t, unsigned long long size, DenseView v,
                                        const unsigned* __restrict__ img) {
  for (unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; i < size;
       i += (unsigned long long)gridDim.x * blockDim.x) {
    DenseSlot& e = t[i];
    if (e.key == DENSE_EMPTY) continue;
    const double c = (double)e.count;
    double r;
    const int pix = dense_pixel(v, e.sum[0] / c, e.sum[1] / c, e.sum[2] / c, r);
    const unsigned b = img[pix];
    if (b < 0x7f800000u && (double)__uint_as_float(b) > r + v.margin) e.evidence = dense_add_miss(e.evidence);
  }
}

// ---- 8^3-brick index: carve mode's live occupancy index and the target's ray index
// An open-addressing hash of brick keys (dense_hash, linear probe, load factor <= 0.5) with each brick's 512-bit mask
// of occupied voxels; brick key and bit come from the key codec.  The ray index also keeps, per slot, the sorted
// position of its brick's first voxel (base) and, per sorted position, a target index (idx); the live index has neither.
constexpr int DENSE_BRICK_WORDS = 8;                 // 64-bit words of a brick's mask

struct DenseBrickIndex {                    // device view, by value in the kernel arguments
  unsigned long long* key = nullptr;        // brick key per slot, DENSE_EMPTY when free; null: no index
  unsigned long long* mask = nullptr;       // DENSE_BRICK_WORDS words per slot
  unsigned long long slots_mask = 0;        // slots - 1 (a power of two)
  unsigned* base = nullptr;                 // ray index: per slot, sorted position of the brick's first voxel
  int* idx = nullptr;                       // ray index: per sorted position, target index

  __host__ __device__ unsigned long long slots() const { return key ? slots_mask + 1 : 0; }

  // the slot of `brick`; when absent, -1 (find) or a slot claimed for it, with *claimed set (find_or_claim)
  template <bool CLAIM>
  __device__ __forceinline__ long long probe(unsigned long long brick, bool* claimed) const {
    unsigned long long h = dense_hash(brick) & slots_mask;
    for (;;) {
      const unsigned long long k = CLAIM ? atomicCAS(&key[h], DENSE_EMPTY, brick) : __ldg(&key[h]);
      if (k == brick) return (long long)h;
      if (k == DENSE_EMPTY) {
        if (!CLAIM) return -1;
        if (claimed) *claimed = true;
        return (long long)h;
      }
      h = (h + 1) & slots_mask;
    }
  }
  __device__ __forceinline__ long long find(unsigned long long brick) const { return probe<false>(brick, nullptr); }
  __device__ __forceinline__ long long find_or_claim(unsigned long long b, bool* claimed = nullptr) const {
    return probe<true>(b, claimed);
  }
  __device__ __forceinline__ void set(long long slot, unsigned bit) const {
    atomicOr(&mask[slot * DENSE_BRICK_WORDS + (bit >> 6)], 1ull << (bit & 63));
  }
  __device__ __forceinline__ unsigned long long word(long long slot, unsigned bit) const {
    return __ldg(&mask[slot * DENSE_BRICK_WORDS + (bit >> 6)]);
  }
  __device__ __forceinline__ bool test(long long slot, unsigned bit) const {
    return (word(slot, bit) >> (bit & 63)) & 1ull;
  }
};

// ---- ray casting the target (include/loam_b200.h "loam_b200_dense_raycast")
// Ray index: built from the target's keys: composite key brick << 9 | bit, sorted (dense_sort64), so each brick's
// voxels are one run in bit order; idx[j] = the target index of sorted position j, and a brick's slot keeps its mask
// and the position of its run's head.  A voxel's target index is then idx[base + popc(mask below its bit)].
constexpr int DENSE_RAY_MAX_STEPS = 3 * 65536 + 4;   // max_range / leaf <= 65536 crosses at most sqrt(3) 65536 + 3 faces

struct DenseRayArgs {                  // by value in the kernel arguments
  double ox, oy, oz;                   // origin: the pose's float pos
  double cx, sx, cy, sy, cz, sz;       // std::cos / std::sin of the pose's float rot_x, rot_y, rot_z (host)
  double leaf, min_range, max_range;
};

__device__ __forceinline__ unsigned long long dense_brick_composite(unsigned long long key) {
  int ux, uy, uz;
  dense_unpack(key, ux, uy, uz);
  return (dense_brick(ux, uy, uz) << 9) | dense_brick_bit(ux, uy, uz);
}

// composite keys of the target's voxels + the (low word, index) pairs of the first sort pass
__global__ void dense_brick_key_kernel(const unsigned long long* __restrict__ keys, int n,
                                       unsigned long long* __restrict__ comp, unsigned* __restrict__ keys_lo,
                                       int* __restrict__ vals) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const unsigned long long c = dense_brick_composite(keys[i]);
  comp[i] = c;
  keys_lo[i] = (unsigned)c;
  vals[i] = i;
}

// per sorted position: keep the target index, count the bricks (run heads)
__global__ void dense_brick_count_kernel(const unsigned long long* __restrict__ comp, const int* __restrict__ order,
                                         int n, int* __restrict__ idx, int* __restrict__ bricks) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const int o = order[j];
  idx[j] = o;
  if (j == 0 || (comp[o] >> 9) != (comp[order[j - 1]] >> 9)) atomicAdd(bricks, 1);
}

// per sorted position: find or claim the brick's slot, set the voxel's bit; the head sets base
__global__ void dense_brick_fill_kernel(const unsigned long long* __restrict__ comp, int n, DenseBrickIndex ix) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const unsigned long long c = comp[ix.idx[j]], brick = c >> 9;
  const long long h = ix.find_or_claim(brick);
  ix.set(h, (unsigned)(c & 511));
  if (j == 0 || (comp[ix.idx[j - 1]] >> 9) != brick) ix.base[h] = (unsigned)j;
}

// The voxel walk of a ray from o along d (Amanatides-Woo) through a brick index, shared by the ray cast and carve mode,
// fp64 without FMA: start voxel floor(o_a / L); per axis with d_a != 0 inv_a = 1 / d_a and t_next_a = ((double)k * L -
// o_a) * inv_a with k = v_a + 1 (d_a > 0) or v_a (d_a < 0); +inf when d_a == 0.  The current voxel spans [t_enter,
// t_exit = min t_next); step() moves along axis() -- the smallest t_next, ties x, y, z -- and recomputes only that
// axis's t_next, from its new index, so no error accumulates.  The walk keeps `slot`, the current voxel's brick in the
// index it walks: probed at the start and again only when a step enters another 8^3 brick.
struct DenseWalk {
  double ox, oy, oz, L, ivx, ivy, ivz, tnx, tny, tnz;
  int vx, vy, vz, stx, sty, stz;
  long long slot;  // -1 when the brick is empty or the voxel outside the key range

  __device__ __forceinline__ DenseWalk(const DenseBrickIndex& ix, double ox_, double oy_, double oz_, double dx,
                                       double dy, double dz, double L_)
      : ox(ox_), oy(oy_), oz(oz_), L(L_) {
    const double inf = __longlong_as_double(0x7ff0000000000000ll);
    vx = (int)floor(ox / L);
    vy = (int)floor(oy / L);
    vz = (int)floor(oz / L);
    stx = dx > 0.0 ? 1 : -1;
    sty = dy > 0.0 ? 1 : -1;
    stz = dz > 0.0 ? 1 : -1;
    ivx = 1.0 / dx;
    ivy = 1.0 / dy;
    ivz = 1.0 / dz;
    tnx = dx != 0.0 ? ((double)(dx > 0.0 ? vx + 1 : vx) * L - ox) * ivx : inf;
    tny = dy != 0.0 ? ((double)(dy > 0.0 ? vy + 1 : vy) * L - oy) * ivy : inf;
    tnz = dz != 0.0 ? ((double)(dz > 0.0 ? vz + 1 : vz) * L - oz) * ivz : inf;
    slot = brick(ix);
  }
  __device__ __forceinline__ int axis() const { return (tnx <= tny && tnx <= tnz) ? 0 : (tny <= tnz ? 1 : 2); }
  __device__ __forceinline__ double t_next(int ax) const { return ax == 0 ? tnx : (ax == 1 ? tny : tnz); }
  __device__ __forceinline__ void step(const DenseBrickIndex& ix, int ax) {
    if (advance(ax)) slot = brick(ix);
  }
  // the current voxel's bit in its brick
  __device__ __forceinline__ unsigned bit() const {
    return dense_brick_bit(vx + DENSE_KEY_BIAS, vy + DENSE_KEY_BIAS, vz + DENSE_KEY_BIAS);
  }

 private:
  // one step along `ax`: whether it entered another brick
  __device__ __forceinline__ bool advance(int ax) {
    if (ax == 0) {
      vx += stx;
      tnx = ((double)(stx > 0 ? vx + 1 : vx) * L - ox) * ivx;
      return ((vx + DENSE_KEY_BIAS) & 7) == (stx > 0 ? 0 : 7);
    }
    if (ax == 1) {
      vy += sty;
      tny = ((double)(sty > 0 ? vy + 1 : vy) * L - oy) * ivy;
      return ((vy + DENSE_KEY_BIAS) & 7) == (sty > 0 ? 0 : 7);
    }
    vz += stz;
    tnz = ((double)(stz > 0 ? vz + 1 : vz) * L - oz) * ivz;
    return ((vz + DENSE_KEY_BIAS) & 7) == (stz > 0 ? 0 : 7);
  }
  __device__ __forceinline__ long long brick(const DenseBrickIndex& ix) const {
    if (vx < -DENSE_KEY_BIAS || vx >= DENSE_KEY_BIAS || vy < -DENSE_KEY_BIAS || vy >= DENSE_KEY_BIAS ||
        vz < -DENSE_KEY_BIAS || vz >= DENSE_KEY_BIAS)
      return -1;
    return ix.find(dense_brick(vx + DENSE_KEY_BIAS, vy + DENSE_KEY_BIAS, vz + DENSE_KEY_BIAS));
  }
};

// One thread per ray (tests/raycast_reference.py restates it), fp64 without FMA, each operation rounded on its own:
//   |p| = sqrt((x*x + y*y) + z*z) of the float components; u = p / |p|; d = rotZ, rotX, rotY of u (to_map64's order);
//   a non-finite or zero p has no hit.  The walk is DenseWalk's.
//   Per voxel [t_enter, t_exit = min t_next): stop when t_enter > max_range; the first occupied voxel with
//   t_exit > min_range is the hit, at t = clamp(num / den, lo, hi) on its surfel (den != 0) or lo (no normal, or
//   den == 0), lo = max(t_enter, min_range), hi = t_exit; t > max_range is no hit.  Then one step along the axis of the
//   smallest t_next (ties x, y, z); t_enter = its old t_next; only its t_next is recomputed, from the new index.
// dense_ray_hit is the walk and hit from origin (ox, oy, oz) along the map-frame unit d: the hit's target index and *t,
// or -1.  It is the one copy of the rule; dense_raycast_kernel and dense_place_build_kernel both run it.
__device__ __forceinline__ int dense_ray_hit(const DenseBrickIndex& ix, const float4* __restrict__ cent,
                                             const float4* __restrict__ nrm, double ox, double oy, double oz, double dx,
                                             double dy, double dz, double leaf, double min_range, double max_range,
                                             double* t_out) {
  DenseWalk w(ix, ox, oy, oz, dx, dy, dz, leaf);
  double t_enter = 0.0, lo = 0.0, hi = 0.0;
  int j_hit = -1;
  for (int s = 0; s < DENSE_RAY_MAX_STEPS; s++) {
    if (t_enter > max_range) break;
    const int ax = w.axis();
    const double t_exit = w.t_next(ax);
    if (w.slot >= 0 && t_exit > min_range) {
      const unsigned bit = w.bit();
      if (ix.test(w.slot, bit)) {  // its target index: the brick's voxels below it, after the brick's base
        const unsigned long long* m = ix.mask + w.slot * DENSE_BRICK_WORDS;
        int below = __popcll(ix.word(w.slot, bit) & ((1ull << (bit & 63)) - 1ull));
        for (unsigned k = 0; k < (bit >> 6); k++) below += __popcll(__ldg(&m[k]));
        j_hit = __ldg(&ix.idx[__ldg(&ix.base[w.slot]) + below]);
        lo = t_enter > min_range ? t_enter : min_range;
        hi = t_exit;
        break;
      }
    }
    t_enter = t_exit;
    w.step(ix, ax);
  }
  if (j_hit < 0) return -1;
  double t = lo;  // the surfel range, outside the walk (its division stays out of the loop)
  const float4 nv = nrm[j_hit];
  if (!isnan(nv.x)) {
    const double den = ((double)nv.x * dx + (double)nv.y * dy) + (double)nv.z * dz;
    if (den != 0.0) {
      const float4 c = cent[j_hit];
      const double num = ((double)nv.x * ((double)c.x - ox) + (double)nv.y * ((double)c.y - oy)) +
                         (double)nv.z * ((double)c.z - oz);
      const double q = num / den;
      t = q < lo ? lo : (q > hi ? hi : q);
    }
  }
  if (t > max_range) return -1;
  *t_out = t;
  return j_hit;
}

__global__ void
dense_raycast_kernel(const float4* __restrict__ rays, int n, DenseRayArgs a, DenseBrickIndex ix,
                     const float4* __restrict__ cent, const float4* __restrict__ nrm, float* __restrict__ range,
                     int* __restrict__ index) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float4 p = rays[i];
  const double px = (double)p.x, py = (double)p.y, pz = (double)p.z;
  const double len = sqrt((px * px + py * py) + pz * pz);
  if (isfinite(p.x) && isfinite(p.y) && isfinite(p.z) && len > 0.0) {
    const double ux = px / len, uy = py / len, uz = pz / len;
    const double x1 = a.cz * ux - a.sz * uy, y1 = a.sz * ux + a.cz * uy;
    const double y2 = a.cx * y1 - a.sx * uz, z2 = a.sx * y1 + a.cx * uz;
    const double dx = a.cy * x1 + a.sy * z2, dy = y2, dz = a.cy * z2 - a.sy * x1;
    double t;
    const int j_hit = dense_ray_hit(ix, cent, nrm, a.ox, a.oy, a.oz, dx, dy, dz, a.leaf, a.min_range, a.max_range, &t);
    if (j_hit >= 0) {
      range[i] = (float)t;
      index[i] = j_hit;
      return;
    }
  }
  range[i] = __int_as_float(0x7f800000);  // no hit
  index[i] = -1;
}

// ---- distance field of the target (include/loam_b200.h "Distance field of the whole-run voxel map")
// Exact squared EDT in voxel units over the padded box (the box grown by pad = floor(max_distance / L) + 1 voxels on
// every side), separable: x pass (nearest site on each x line, fused with the rasterisation from the ray index), then
// Meijster's integer lower envelope along y and along z.  Values stay below 3 * 8191^2 < 2^31, so int32 holds every
// one; DENSE_EDT_INF marks "no site on this line" and never enters a sum.  The y pass only runs the lines whose x lies
// in the box, and the z pass only those whose x and y do, each writing only the positions inside the box: the rest
// of the padded box is only ever a source of sites.
constexpr int DENSE_EDT_INF = 0x7fffffff;
constexpr int DENSE_EDT_MAX_RATIO = 1024;        // max_distance / leaf
constexpr int DENSE_EDT_MAX_AXIS = 8192;         // padded cells per axis
constexpr long long DENSE_EDT_MAX_CELLS = 1ll << 27;  // padded cells
constexpr int DENSE_EDT_LINE_THREADS = 128;

struct DenseDistArgs {  // by value in the kernel arguments
  double L, max_distance;
  int lo[3], n[3];      // the box: first voxel and cells per axis
};

// x pass, one warp per padded x line (y, z): a lane per cell of each 32-cell chunk probes its brick and tests the bit;
// a warp max scan carries the nearest site at or left of x forwards, then a min scan the nearest at or right of x
// backwards.  g = the squared distance to the nearer, DENSE_EDT_INF without a site on the line.  The forward pass
// leaves the left site's index in g, which the backward pass (same lane, same cell) reads back.
__global__ void __launch_bounds__(256) dense_edt_x_kernel(DenseBrickIndex ix, int plx, int ply, int plz, int nxp,
                                                          int nyp, long long lines, int* __restrict__ g) {
  const long long line = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (line >= lines) return;  // whole warps
  const int uy = ply + (int)(line % nyp) + DENSE_KEY_BIAS, uz = plz + (int)(line / nyp) + DENSE_KEY_BIAS;
  int* row = g + line * nxp;
  int carry = -1;  // the nearest site so far, -1: none
  for (int x0 = 0; x0 < nxp; x0 += 32) {
    const int x = x0 + lane;
    bool occ = false;
    if (x < nxp) {
      const int ux = plx + x + DENSE_KEY_BIAS;
      const long long slot = ix.find(dense_brick(ux, uy, uz));
      occ = slot >= 0 && ix.test(slot, dense_brick_bit(ux, uy, uz));
    }
    int v = occ ? x : -1;
    for (int o = 1; o < 32; o <<= 1) {
      const int u = __shfl_up_sync(0xffffffffu, v, o);
      if (lane >= o) v = max(v, u);
    }
    v = max(v, carry);
    if (x < nxp) row[x] = v;
    carry = __shfl_sync(0xffffffffu, v, 31);
  }
  carry = DENSE_EDT_INF;
  for (int x0 = (nxp - 1) & ~31; x0 >= 0; x0 -= 32) {
    const int x = x0 + lane;
    const int left = x < nxp ? row[x] : -1;
    int v = left == x ? x : DENSE_EDT_INF;
    for (int o = 1; o < 32; o <<= 1) {
      const int u = __shfl_down_sync(0xffffffffu, v, o);
      if (lane + o < 32) v = min(v, u);
    }
    v = min(v, carry);
    if (x < nxp) {
      const int d = min(left >= 0 ? x - left : DENSE_EDT_INF, v != DENSE_EDT_INF ? v - x : DENSE_EDT_INF);
      row[x] = d == DENSE_EDT_INF ? DENSE_EDT_INF : d * d;
    }
    carry = __shfl_sync(0xffffffffu, v, 0);
  }
}

// Meijster's lower envelope of the parabolas (u - s)^2 + f(s) of one line's finite sites, its stacks s, t (the first
// position where s is the lowest) and f(s) in global scratch at stride `ss` (consecutive threads: consecutive x, so
// every access is coalesced); the top stays in registers.  Sep is the floor division of (u^2 - s^2 + f(u) - f(s)) by
// 2 (u - s) in int64.  Ties keep the earlier site (only values are ever read).
struct DenseEdtEnvelope {
  int* S;
  int* T;
  int* G;
  long long ss;
  int q = -1, s = 0, t = 0, gs = 0;  // top of the stacks, q == -1: no site

  __device__ __forceinline__ void load() {
    s = S[q * ss];
    t = T[q * ss];
    gs = G[q * ss];
  }
  __device__ __forceinline__ void push(int u, int w, int gu) {
    q++;
    s = u;
    t = w;
    gs = gu;
    S[q * ss] = u;
    T[q * ss] = w;
    G[q * ss] = gu;
  }
  // the envelope of f[0], f[fs], ... f[(m - 1) fs]
  __device__ __forceinline__ void build(const int* __restrict__ f, long long fs, int m) {
    for (int u = 0; u < m; u++) {
      const int gu = f[u * fs];
      if (gu == DENSE_EDT_INF) continue;
      while (q >= 0) {
        const long long a = (long long)(t - s) * (t - s) + gs, b = (long long)(t - u) * (t - u) + gu;
        if (a <= b) break;
        if (--q >= 0) load();
      }
      if (q < 0) {
        push(u, 0, gu);
        continue;
      }
      const long long num = ((long long)u * u - (long long)s * s) + ((long long)gu - gs), den = 2ll * (u - s);
      const long long w = (num >= 0 ? num / den : -((-num + den - 1) / den)) + 1;
      if (w < m) push(u, (int)w, gu);
    }
  }
  // the lower envelope at u, for u descending from the end of the line (DENSE_EDT_INF without sites)
  __device__ __forceinline__ int at(int u) {
    if (q < 0) return DENSE_EDT_INF;
    while (t > u) {
      q--;
      load();
    }
    return (u - s) * (u - s) + gs;
  }
};

// y pass: one thread per line (x, z) with x in the box and z in the padded box; reads the x pass (padded layout),
// writes the positions y in the box of b[(z, y, x)] (layout nx x ny x nzp)
__global__ void __launch_bounds__(DENSE_EDT_LINE_THREADS)
dense_edt_y_kernel(const int* __restrict__ g, int pad, int nx, int ny, int nxp, int nyp, int nzp, int* __restrict__ b,
                   int* S, int* T, int* G) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= (long long)nx * nzp) return;
  const int x = (int)(i % nx), z = (int)(i / nx);
  const long long base = (long long)z * nyp * nx + x;  // the line's stacks: [z][position][x]
  DenseEdtEnvelope e{S + base, T + base, G + base, nx};
  e.build(g + (long long)z * nyp * nxp + pad + x, nxp, nyp);
  int* out = b + (long long)z * ny * nx + x;
  for (int y = ny - 1; y >= 0; y--) out[(long long)y * nx] = e.at(pad + y);
}

// z pass: one thread per line (x, y) of the box; reads the y pass, writes the field: sq (-1 beyond) and, with `dist`,
// the float distance
__global__ void __launch_bounds__(DENSE_EDT_LINE_THREADS)
dense_edt_z_kernel(const int* __restrict__ b, int pad, DenseDistArgs a, int nzp, int* S, int* T, int* G,
                   int* __restrict__ sq, float* __restrict__ dist) {
  const int nx = a.n[0], ny = a.n[1], nz = a.n[2];
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x, plane = (long long)nx * ny;
  if (i >= plane) return;
  DenseEdtEnvelope e{S + i, T + i, G + i, plane};  // stacks: [position][y][x]
  e.build(b + i, plane, nzp);
  for (int z = nz - 1; z >= 0; z--) {
    const int v = e.at(pad + z);
    const double w = v == DENSE_EDT_INF ? 0.0 : sqrt((double)v) * a.L;
    const bool beyond = v == DENSE_EDT_INF || w > a.max_distance;
    sq[z * plane + i] = beyond ? -1 : v;
    if (dist) dist[z * plane + i] = beyond ? __int_as_float(0x7f800000) : (float)w;
  }
}

// Distance query, one thread per point, fp64 without FMA, each operation rounded on its own (the header states the
// expression order): trilinear in the corner distances along x, then y, then z; the gradient per axis the same lerps
// of the corner differences along that axis, divided by L.  NaN outside the hull of the cell centres.
__device__ __forceinline__ double dense_lerp(double a, double b, double f) { return a + f * (b - a); }

__global__ void dense_distance_query_kernel(const float4* __restrict__ p, int n, DenseDistArgs a,
                                            const int* __restrict__ sq, float* __restrict__ dist,
                                            float* __restrict__ grad) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  const float4 q = p[k];
  const double c[3] = {(double)q.x, (double)q.y, (double)q.z};
  int i[3];
  double f[3];
  bool ok = true;
#pragma unroll
  for (int ax = 0; ax < 3; ax++) {
    const double g = (c[ax] / a.L - 0.5) - (double)a.lo[ax];
    ok = ok && a.n[ax] >= 2 && g >= 0.0 && g <= (double)(a.n[ax] - 1);
    i[ax] = ok ? min((int)floor(g), a.n[ax] - 2) : 0;
    f[ax] = g - (double)i[ax];
  }
  if (!ok) {
    const float nan = __int_as_float(0x7fffffff);
    dist[k] = nan;
    if (grad) grad[3 * k] = grad[3 * k + 1] = grad[3 * k + 2] = nan;
    return;
  }
  const long long sy = a.n[0], sz = (long long)a.n[0] * a.n[1];
  const long long o = (long long)i[2] * sz + (long long)i[1] * sy + i[0];
  double w[8];  // w[z * 4 + y * 2 + x]
#pragma unroll
  for (int j = 0; j < 8; j++) {
    const int v = __ldg(&sq[o + ((j >> 2) & 1) * sz + ((j >> 1) & 1) * sy + (j & 1)]);
    w[j] = v < 0 ? a.max_distance : sqrt((double)v) * a.L;
  }
  const double fx = f[0], fy = f[1], fz = f[2];
  const double x00 = dense_lerp(w[0], w[1], fx), x10 = dense_lerp(w[2], w[3], fx);
  const double x01 = dense_lerp(w[4], w[5], fx), x11 = dense_lerp(w[6], w[7], fx);
  dist[k] = (float)dense_lerp(dense_lerp(x00, x10, fy), dense_lerp(x01, x11, fy), fz);
  if (!grad) return;
  const double gx = dense_lerp(dense_lerp(w[1] - w[0], w[3] - w[2], fy), dense_lerp(w[5] - w[4], w[7] - w[6], fy), fz);
  const double gy = dense_lerp(dense_lerp(w[2] - w[0], w[3] - w[1], fx), dense_lerp(w[6] - w[4], w[7] - w[5], fx), fz);
  const double gz = dense_lerp(dense_lerp(w[4] - w[0], w[5] - w[1], fx), dense_lerp(w[6] - w[2], w[7] - w[3], fx), fy);
  grad[3 * k] = (float)(gx / a.L);
  grad[3 * k + 1] = (float)(gy / a.L);
  grad[3 * k + 2] = (float)(gz / a.L);
}

// ---- place descriptors and global relocalisation (include/loam_b200.h "Place recognition")
// Polar height descriptor, rings x sectors cells (ring-major), each the float bits of the largest value v > 0 of its
// points (0: none).  Bits of non-negative floats order like the floats, so atomicMax gives the same cell in any order.
constexpr int DENSE_PLACE_MAX_RINGS = 64;
constexpr int DENSE_PLACE_MAX_SECTORS = 720;
constexpr int DENSE_PLACE_MAX_CELLS = 4096;  // the descriptor of one CTA in shared memory
constexpr int DENSE_PLACE_THREADS = 256;

struct DensePlaceArgs {  // by value in the kernel arguments
  double ring_w;         // max_radius / rings (host, double)
  double max_radius, height_offset;
  int rings, sectors;
};

// The cell of one sensor-frame point and its value's bits, or -1 (fp64 without FMA; tests/place_reference.py restates
// it): a non-finite point, r = sqrt(x*x + z*z) == 0 or r >= max_radius, or v = (float)(y + height_offset) not in
// (0, FLT_MAX] has none.  ring = min(floor(r / ring_w), rings - 1).  Sector: the number of boundaries k in
// [1, sectors) the point is at or past, past(k) = h_p > h_k, or h_p == h_k and x * tab[k].x - z * tab[k].y >= 0, with
// h_k = (2k >= sectors), h_p = 0 when x > 0 or (x == 0 and z > 0), else 1; tab[k] = (cos, sin) of k D, the boundary
// at pi exactly (-1, 0).  past() holds on a prefix of the boundaries (they lie at least 0.5 deg apart, far beyond
// the rounding of the test, and no point of a half is antipodal to a boundary of its half), so bisection finds the
// count.
__device__ __forceinline__ int dense_place_cell(const DensePlaceArgs& pa, const double2* __restrict__ tab, float fx,
                                                float fy, float fz, unsigned* bits) {
  if (!(isfinite(fx) && isfinite(fy) && isfinite(fz))) return -1;
  const double x = (double)fx, y = (double)fy, z = (double)fz;
  const double r = sqrt(x * x + z * z);
  if (r == 0.0 || !(r < pa.max_radius)) return -1;
  const float v = (float)(y + pa.height_offset);
  if (!(v > 0.f && v <= 3.402823466e38f)) return -1;
  int ring = (int)floor(r / pa.ring_w);
  if (ring > pa.rings - 1) ring = pa.rings - 1;
  const int hp = (x > 0.0 || (x == 0.0 && z > 0.0)) ? 0 : 1;
  int lo = 1, hi = pa.sectors;  // past(k) for every k < lo, !past(k) for every k >= hi
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    const double2 cs = __ldg(&tab[mid]);
    const int hk = 2 * mid >= pa.sectors ? 1 : 0;
    if (hp > hk || (hp == hk && x * cs.x - z * cs.y >= 0.0)) lo = mid + 1;
    else hi = mid;
  }
  *bits = __float_as_uint(v);
  return ring * pa.sectors + (lo - 1);
}

// the CTA's descriptor (shared, zeroed by the caller) -> atomicMax into the global one
__device__ __forceinline__ void dense_place_flush(const unsigned* s_desc, unsigned* __restrict__ desc, int cells) {
  __syncthreads();
  for (int k = threadIdx.x; k < cells; k += blockDim.x)
    if (s_desc[k]) atomicMax(&desc[k], s_desc[k]);
}

__device__ __forceinline__ void dense_place_zero(unsigned* s_desc, int cells) {
  for (int k = threadIdx.x; k < cells; k += blockDim.x) s_desc[k] = 0u;
  __syncthreads();
}

// query: one thread per point into the CTA's descriptor, then one flush per CTA (desc zeroed before the launch)
__global__ void __launch_bounds__(DENSE_PLACE_THREADS)
dense_place_bin_kernel(const float4* __restrict__ p, int n, DensePlaceArgs pa, const double2* __restrict__ tab,
                       unsigned* __restrict__ desc) {
  __shared__ unsigned s_desc[DENSE_PLACE_MAX_CELLS];
  const int cells = pa.rings * pa.sectors;
  dense_place_zero(s_desc, cells);
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    const float4 q = p[i];
    unsigned b;
    const int cell = dense_place_cell(pa, tab, q.x, q.y, q.z, &b);
    if (cell >= 0) atomicMax(&s_desc[cell], b);
  }
  dense_place_flush(s_desc, desc, cells);
}

// database: blockIdx.y = candidate c0 + y, one thread per ray (dense_raycast_kernel's u and dense_ray_hit from the
// candidate's float position with rot = 0, so d = u), the hit's point (float)((double)(float)t * u_a) per axis binned
// by dense_place_cell; desc (zeroed before the launch) holds one descriptor per candidate
__global__ void __launch_bounds__(DENSE_PLACE_THREADS)
dense_place_build_kernel(const float4* __restrict__ rays, int n, const float* __restrict__ pos, int c0, DenseRayArgs a,
                         DenseBrickIndex ix, const float4* __restrict__ cent, const float4* __restrict__ nrm,
                         DensePlaceArgs pa, const double2* __restrict__ tab, unsigned* __restrict__ desc) {
  __shared__ unsigned s_desc[DENSE_PLACE_MAX_CELLS];
  const int cells = pa.rings * pa.sectors;
  const int c = c0 + (int)blockIdx.y;
  dense_place_zero(s_desc, cells);
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    const float4 p = rays[i];
    const double px = (double)p.x, py = (double)p.y, pz = (double)p.z;
    const double len = sqrt((px * px + py * py) + pz * pz);
    if (isfinite(p.x) && isfinite(p.y) && isfinite(p.z) && len > 0.0) {
      const double ux = px / len, uy = py / len, uz = pz / len;
      double t;
      const int j = dense_ray_hit(ix, cent, nrm, (double)pos[3 * c], (double)pos[3 * c + 1], (double)pos[3 * c + 2],
                                  ux, uy, uz, a.leaf, a.min_range, a.max_range, &t);
      if (j >= 0) {
        const double tf = (double)(float)t;
        unsigned b;
        const int cell = dense_place_cell(pa, tab, (float)(tf * ux), (float)(tf * uy), (float)(tf * uz), &b);
        if (cell >= 0) atomicMax(&s_desc[cell], b);
      }
    }
  }
  dense_place_flush(s_desc, desc + (size_t)c * cells, cells);
}

// One CTA per candidate (blockIdx.x), one thread per shift s (strided): columns j ascending, query column j against
// candidate column (j + s) mod sectors; qq, dd and dot are fp64 sums in ascending ring; a column with qq == 0 or
// dd == 0 is skipped, otherwise sim = dot / (sqrt(qq) * sqrt(dd)) is added; dist = 1 - sum / counted, +inf when none.
// The best shift: smallest dist, ties to the smaller s (each thread scans its shifts ascending with a strict <, then
// a tree over (dist, s) pairs).
__global__ void __launch_bounds__(DENSE_PLACE_THREADS)
dense_place_match_kernel(const unsigned* __restrict__ db, const unsigned* __restrict__ query, int rings, int sectors,
                         double* __restrict__ best_dist, int* __restrict__ best_shift) {
  __shared__ float s_q[DENSE_PLACE_MAX_CELLS], s_d[DENSE_PLACE_MAX_CELLS];
  __shared__ double s_qn[DENSE_PLACE_MAX_SECTORS], s_dn[DENSE_PLACE_MAX_SECTORS];
  __shared__ double s_bd[DENSE_PLACE_THREADS];
  __shared__ int s_bs[DENSE_PLACE_THREADS];
  const int cells = rings * sectors;
  const unsigned* d = db + (size_t)blockIdx.x * cells;
  for (int k = threadIdx.x; k < cells; k += blockDim.x) {
    s_q[k] = __uint_as_float(__ldg(&query[k]));
    s_d[k] = __uint_as_float(__ldg(&d[k]));
  }
  __syncthreads();
  for (int j = threadIdx.x; j < sectors; j += blockDim.x) {
    double qq = 0.0, dd = 0.0;
    for (int r = 0; r < rings; r++) {
      const double q = (double)s_q[r * sectors + j], e = (double)s_d[r * sectors + j];
      qq += q * q;
      dd += e * e;
    }
    s_qn[j] = sqrt(qq);  // a positive sum of squares of floats is far above the smallest double: zero iff qq == 0
    s_dn[j] = sqrt(dd);
  }
  __syncthreads();
  double bd = __longlong_as_double(0x7ff0000000000000ll);
  int bs = sectors;
  for (int s = threadIdx.x; s < sectors; s += blockDim.x) {
    double sum = 0.0;
    int counted = 0;
    for (int j = 0; j < sectors; j++) {
      int jj = j + s;
      if (jj >= sectors) jj -= sectors;
      if (s_qn[j] == 0.0 || s_dn[jj] == 0.0) continue;
      double dot = 0.0;
      for (int r = 0; r < rings; r++) dot += (double)s_q[r * sectors + j] * (double)s_d[r * sectors + jj];
      sum += dot / (s_qn[j] * s_dn[jj]);
      counted++;
    }
    const double dist = counted ? 1.0 - sum / (double)counted : __longlong_as_double(0x7ff0000000000000ll);
    if (dist < bd || bs == sectors) {
      bd = dist;
      bs = s;
    }
  }
  s_bd[threadIdx.x] = bd;
  s_bs[threadIdx.x] = bs;
  __syncthreads();
  for (int o = DENSE_PLACE_THREADS / 2; o > 0; o >>= 1) {
    if (threadIdx.x < o) {
      const double d2 = s_bd[threadIdx.x + o];
      const int s2 = s_bs[threadIdx.x + o];
      if (d2 < s_bd[threadIdx.x] || (d2 == s_bd[threadIdx.x] && s2 < s_bs[threadIdx.x])) {
        s_bd[threadIdx.x] = d2;
        s_bs[threadIdx.x] = s2;
      }
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    best_dist[blockIdx.x] = s_bd[0];
    best_shift[blockIdx.x] = s_bs[0];
  }
}

// ---- carve mode of the visibility pass (include/loam_b200.h "loam_b200_dense_carving")
// Live occupancy index: a DenseBrickIndex over the live table without base or idx (keys and masks only, so a rehash of
// the voxel table leaves it valid).  Built from the table when carve mode is switched on, then kept current by the
// insertion (dense_live_insert_kernel sets the bits of the voxels it admits); it grows like the table, from a host-side
// bound of its bricks, with a rehash on the device.  ctr->bricks counts the claimed bricks, so the host can tighten
// that bound from the counters each insertion mirrors.

// set voxel `key`'s bit: find or claim its brick (a claim counts a brick)
__device__ __forceinline__ void dense_live_set(const DenseBrickIndex& ix, unsigned long long key,
                                               DenseCounters* __restrict__ ctr) {
  const unsigned long long c = dense_brick_composite(key);
  bool claimed = false;
  const long long h = ix.find_or_claim(c >> 9, &claimed);
  if (claimed) atomicAdd(&ctr->bricks, 1ull);
  ix.set(h, (unsigned)(c & 511));
}

// build: one thread per table slot (carve mode switched on with voxels stored; never on the per-sweep path)
__global__ void dense_live_build_kernel(const DenseSlot* __restrict__ t, unsigned long long size, DenseBrickIndex ix,
                                        DenseCounters* __restrict__ ctr) {
  const unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x;
  if (i >= size) return;
  const unsigned long long k = t[i].key;
  if (k != DENSE_EMPTY) dense_live_set(ix, k, ctr);
}

// growth: every brick of the old index moves to the new one with its mask (each brick once)
__global__ void dense_live_rehash_kernel(DenseBrickIndex old, DenseBrickIndex ix) {
  const unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x;
  if (i > old.slots_mask) return;
  const unsigned long long b = old.key[i];
  if (b == DENSE_EMPTY) return;
  const long long h = ix.find_or_claim(b);
#pragma unroll
  for (int w = 0; w < DENSE_BRICK_WORDS; w++) ix.mask[h * DENSE_BRICK_WORDS + w] = old.mask[i * DENSE_BRICK_WORDS + w];
}

// in the insertion, between dense_insert_kernel and dense_finish_kernel: the voxels that kernel admitted (new runs
// ranked below the room, the same test on the same ctr->voxels) get their bits
__global__ void dense_live_insert_kernel(DenseRuns runs, const int* __restrict__ n_runs, const unsigned* __restrict__ rank,
                                         const unsigned* __restrict__ block_off, DenseBrickIndex ix,
                                         DenseCounters* __restrict__ ctr, unsigned long long max_voxels) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= *n_runs || runs.slot[r] != -1) return;
  const unsigned long long nr = rank[r] + block_off[r / SCAN_BS];
  if (ctr->voxels + nr >= max_voxels) return;
  dense_live_set(ix, runs.key[r], ctr);
}

// Misses of one pass without a pass over the table: stamp[s] (one word per table slot) holds 2e when slot s is in K
// for pass e and 2e + 1 once a ray of pass e has carved it; stale words from earlier passes match neither.
struct DenseCarveArgs {                // by value in the kernel arguments
  double ox, oy, oz;                   // origin: the pose's float pos
  double leaf, margin, max_range;
  unsigned k_code, c_code;             // 2e and 2e + 1 of this pass
};

// K: one thread per point, the voxel by the map's rule (dense_key_of); a stored one is stamped "in K"
__global__ void dense_carve_mark_kernel(const float4* __restrict__ p, int n, float inv, const DenseSlot* __restrict__ t,
                                        unsigned long long tmask, unsigned* __restrict__ stamp, unsigned k_code) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const unsigned long long k = dense_key_of(p[i], inv);
  if (k == DENSE_EMPTY) return;
  const long long s = dense_find(t, tmask, k);
  if (s >= 0) stamp[s] = k_code;
}

// One thread per ray (tests/carve_reference.py restates it), fp64 without FMA: e = p - o, r = sqrt((ex*ex + ey*ey) +
// ez*ez), d = e / r (a non-finite p or r == 0 casts nothing); T = min(r - margin, max_range); DenseWalk from o along d
// until the first voxel with t_exit > T; every voxel before it that the index holds is carved, with a table probe only
// for an occupied voxel.  The first ray to carve a slot that is not in K moves its stamp to c_code and adds the pass's
// one miss, so the count depends neither on the thread order nor on how many rays cross the voxel.
__global__ void __launch_bounds__(128)
dense_carve_kernel(const float4* __restrict__ p, int n, DenseCarveArgs a, DenseBrickIndex ix, DenseSlot* t,
                   unsigned long long tmask, unsigned* stamp) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float4 q = p[i];
  if (!(isfinite(q.x) && isfinite(q.y) && isfinite(q.z))) return;
  const double ex = (double)q.x - a.ox, ey = (double)q.y - a.oy, ez = (double)q.z - a.oz;
  const double r = sqrt((ex * ex + ey * ey) + ez * ez);
  if (!(r > 0.0)) return;
  const double rm = r - a.margin;
  const double T = rm < a.max_range ? rm : a.max_range;
  DenseWalk w(ix, a.ox, a.oy, a.oz, ex / r, ey / r, ez / r, a.leaf);
  for (int s = 0; s < DENSE_RAY_MAX_STEPS; s++) {
    const int ax = w.axis();
    if (w.t_next(ax) > T) break;
    if (w.slot >= 0 && ix.test(w.slot, w.bit())) {
      const long long ts = dense_find(t, tmask, dense_key(w.vx, w.vy, w.vz));
      if (ts >= 0) {
        unsigned old = stamp[ts];
        while (old != a.k_code && old != a.c_code) {
          const unsigned prev = atomicCAS(&stamp[ts], old, a.c_code);
          if (prev == old) {
            t[ts].evidence = dense_add_miss(t[ts].evidence);
            break;
          }
          old = prev;
        }
      }
    }
    w.step(ix, ax);
  }
}

// ---- Euclidean segmentation (include/loam_b200.h "Euclidean segmentation of the whole-run voxel map and of clouds")
// Entries: sorted keys skey[0, n) (a cloud's skipped points carry DENSE_EMPTY and sort last) and their positions spos
// in the same order; orig / inv (cloud mode) map sorted position <-> input index, null for a target (identity).  The
// entry index e of sorted position i is orig[i] (cloud) or i (target).
// Union-find over sorted positions (ECL-CC): par[x] <= x always, because a hook puts the larger root under the
// smaller one and path halving only moves a pointer to an ancestor.  So every non-root points to a smaller index and
// the root of a tree is its smallest member: the final roots -- and every label and record derived from them -- are a
// function of the edge set alone, whatever order the threads hook in.  The bit-for-bit tests rely on this.
constexpr int DENSE_SEG_CHUNK = 256;             // members per chunk of the fixed-order fp64 sums
constexpr unsigned DENSE_SEG_NONE = 0xffffffffu;  // sort key of an entry outside every kept segment (sorts last)

// root of x with path halving (L2 loads: other SMs hook concurrently; a stale parent only costs a retry)
__device__ __forceinline__ int dense_seg_find(int* par, int x) {
  int cur = __ldcg(&par[x]);
  if (cur == x) return x;
  int prev = x, next;
  while (cur > (next = __ldcg(&par[cur]))) {
    __stcg(&par[prev], next);
    prev = cur;
    cur = next;
  }
  return cur;
}

// join the components of a and b: hook the larger root under the smaller with atomicCAS; a failed CAS returns the
// node's new parent (smaller), from which the next attempt climbs
__device__ __forceinline__ void dense_seg_unite(int* par, int a, int b) {
  int ra = dense_seg_find(par, a), rb = dense_seg_find(par, b);
  while (ra != rb) {
    if (ra > rb) {
      const int t = ra;
      ra = rb;
      rb = t;
    }
    const int old = atomicCAS(&par[rb], rb, ra);
    if (old == rb) return;
    rb = old;
  }
}

// cloud mode: key, position and index maps in sorted order (order: the stable two-pass key sort)
__global__ void dense_seg_gather_kernel(const unsigned long long* __restrict__ keys64, const int* __restrict__ order,
                                        int n, const float4* __restrict__ p, unsigned long long* __restrict__ skey,
                                        float4* __restrict__ spos, int* __restrict__ orig, int* __restrict__ inv) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int o = order[i];
  skey[i] = keys64[o];
  spos[i] = p[o];
  orig[i] = o;
  inv[o] = i;
}

__global__ void dense_seg_init_kernel(int n, int* __restrict__ par, int* __restrict__ size, int* __restrict__ first,
                                      int* __restrict__ segid) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  par[i] = i;
  size[i] = 0;
  first[i] = 0x7fffffff;
  segid[i] = -1;
}

// One thread per entry: the entries j > i of dense_box_walk at `radius` with d2 = (dx*dx + dy*dy) + dz*dz <= tol2,
// fp64 of the float coordinates without FMA, join i's component.
__global__ void __launch_bounds__(128)
dense_seg_union_kernel(const unsigned long long* __restrict__ skey, const float4* __restrict__ spos, int n, int radius,
                       double tol2, int* par) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const unsigned long long key = skey[i];
  if (key == DENSE_EMPTY) return;
  const float4 pi = spos[i];
  const double px = (double)pi.x, py = (double)pi.y, pz = (double)pi.z;
  dense_box_walk(skey, n, key, radius, [&](int j) {
    if (j <= i) return;
    const float4 pj = spos[j];
    const double dx = px - (double)pj.x, dy = py - (double)pj.y, dz = pz - (double)pj.z;
    if ((dx * dx + dy * dy) + dz * dz <= tol2) dense_seg_unite(par, i, j);
  });
}

// flatten: every entry's root (-1: not an entry); sizes and smallest entry index accumulate on the roots
__global__ void dense_seg_root_kernel(const unsigned long long* __restrict__ skey, int n, const int* __restrict__ orig,
                                      int* par, int* __restrict__ root, int* __restrict__ size, int* __restrict__ first) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (skey[i] == DENSE_EMPTY) {
    root[i] = -1;
    return;
  }
  const int r = dense_seg_find(par, i);
  root[i] = r;
  atomicAdd(&size[r], 1);
  atomicMin(&first[r], orig ? orig[i] : i);
}

// rank keys, one thread per entry index e: a kept root is written at its smallest entry index (keys_lo =
// 0xffffffff - size, vals = root), everything else sorts last.  A stable sort of these 32-bit keys then ranks by size
// descending, ties by smallest entry index ascending.  *kept counts the segments.
__global__ void dense_seg_rank_key_kernel(int n, const int* __restrict__ inv, const int* __restrict__ root,
                                          const int* __restrict__ size, const int* __restrict__ first, int min_size,
                                          int max_size, unsigned* __restrict__ keys_lo, int* __restrict__ vals,
                                          int* __restrict__ kept) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n) return;
  const int r = root[inv ? inv[e] : e];
  unsigned k = DENSE_SEG_NONE;
  if (r >= 0 && first[r] == e && size[r] >= min_size && size[r] <= max_size) {
    k = 0xffffffffu - (unsigned)size[r];
    atomicAdd(kept, 1);
  }
  keys_lo[e] = k;
  vals[e] = r;
}

// ids in ranked order: segid[root] = rank, segroot[rank] = root
__global__ void dense_seg_id_kernel(const unsigned* __restrict__ keys, const int* __restrict__ vals, int n,
                                    int* __restrict__ segid, int* __restrict__ segroot) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n || keys[r] == DENSE_SEG_NONE) return;
  segid[vals[r]] = r;
  segroot[r] = vals[r];
}

// labels in entry order, and the member keys (segment id, in entry order; vals = sorted position) whose stable sort
// groups each segment's members in ascending entry index
__global__ void dense_seg_label_kernel(int n, const int* __restrict__ inv, const int* __restrict__ root,
                                       const int* __restrict__ segid, int* __restrict__ labels,
                                       unsigned* __restrict__ keys_lo, int* __restrict__ vals) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n) return;
  const int i = inv ? inv[e] : e;
  const int r = root[i];
  const int id = r < 0 ? -1 : segid[r];
  labels[e] = id;
  keys_lo[e] = id < 0 ? DENSE_SEG_NONE : (unsigned)id;
  vals[e] = i;
}

// first member position of each segment in the grouped order
__global__ void dense_seg_head_kernel(const unsigned* __restrict__ keys, int n, int* __restrict__ start) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n) return;
  const unsigned id = keys[p];
  if (id != DENSE_SEG_NONE && (p == 0 || keys[p - 1] != id)) start[id] = p;
}

// min / max that keep the earlier value on a tie (strict <, >), so the sign of a zero is that of the first member
// in entry order to reach the extreme
__device__ __forceinline__ void dense_seg_extend(float4& lo, float4& hi, const float4& a, const float4& b) {
  if (a.x < lo.x) lo.x = a.x;
  if (a.y < lo.y) lo.y = a.y;
  if (a.z < lo.z) lo.z = a.z;
  if (b.x > hi.x) hi.x = b.x;
  if (b.y > hi.y) hi.y = b.y;
  if (b.z > hi.z) hi.z = b.z;
}

// one thread per chunk head (every DENSE_SEG_CHUNK-th member of a segment from its first): the chunk's members in
// ascending entry index summed one after the other in fp64 from 0.0, and their float min / max
__global__ void dense_seg_chunk_kernel(const unsigned* __restrict__ keys, const int* __restrict__ vals, int n,
                                       const float4* __restrict__ spos, const int* __restrict__ start,
                                       double4* __restrict__ csum, float4* __restrict__ clo, float4* __restrict__ chi) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n) return;
  const unsigned id = keys[p];
  if (id == DENSE_SEG_NONE || (p - start[id]) % DENSE_SEG_CHUNK) return;
  double sx = 0.0, sy = 0.0, sz = 0.0;
  float4 lo = spos[vals[p]], hi = lo;
  const int end = min(n, p + DENSE_SEG_CHUNK);
  for (int u = p; u < end && keys[u] == id; u++) {
    const float4 q = spos[vals[u]];
    sx += (double)q.x;
    sy += (double)q.y;
    sz += (double)q.z;
    dense_seg_extend(lo, hi, q, q);
  }
  csum[p] = make_double4(sx, sy, sz, 0.0);
  clo[p] = lo;
  chi[p] = hi;
}

// one thread per segment: the chunk sums added in chunk order from 0.0, min / max over the chunks, the record
__global__ void dense_seg_record_kernel(const int* __restrict__ kept, const int* __restrict__ start,
                                        const int* __restrict__ segroot, const int* __restrict__ size,
                                        const int* __restrict__ first, const double4* __restrict__ csum,
                                        const float4* __restrict__ clo, const float4* __restrict__ chi,
                                        loam_b200_segment* __restrict__ out) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= *kept) return;
  const int s = start[r], root = segroot[r], m = size[root];
  double sx = 0.0, sy = 0.0, sz = 0.0;
  float4 lo = clo[s], hi = chi[s];
  for (int p = s; p < s + m; p += DENSE_SEG_CHUNK) {
    const double4 q = csum[p];
    sx += q.x;
    sy += q.y;
    sz += q.z;
    dense_seg_extend(lo, hi, clo[p], chi[p]);
  }
  loam_b200_segment g;
  g.size = m;
  g.first = first[root];
  g.lo[0] = lo.x;
  g.lo[1] = lo.y;
  g.lo[2] = lo.z;
  g.hi[0] = hi.x;
  g.hi[1] = hi.y;
  g.hi[2] = hi.z;
  const double c = (double)m;
  g.centroid[0] = (float)(sx / c);
  g.centroid[1] = (float)(sy / c);
  g.centroid[2] = (float)(sz / c);
  out[r] = g;
}

// ---- ground patches (include/loam_b200.h "Ground of the whole-run voxel map")
// The candidates and the above-ground entries are the target voxels of class 0, compacted in key order by
// compact_count_kernel<0> at limit 1 and radix_scan_kernel; the compaction of sorted keys is sorted, so dense_box_walk
// and the dense_seg_* kernels run on it unchanged, and the entry order (compacted position) is the target order.

// class per target voxel: 0 a candidate (normal_x not NaN, (double)|n_y| >= cos_max, n_w <= max_curv unless
// check_curv is 0; a NaN w fails), 1 not
__global__ void dense_ground_candidate_kernel(const float4* __restrict__ nrm, int n, double cos_max, float max_curv,
                                              int check_curv, unsigned char* __restrict__ cls) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float4 v = nrm[i];
  const bool cand = !isnan(v.x) && (double)fabsf(v.y) >= cos_max && (!check_curv || v.w <= max_curv);
  cls[i] = cand ? 0 : 1;
}

// the selected target voxels at their compacted position: key, centroid, target index
__global__ void dense_ground_compact_kernel(const unsigned long long* __restrict__ skey,
                                            const float4* __restrict__ cent, int n,
                                            const unsigned* __restrict__ local_pos,
                                            const unsigned* __restrict__ block_off, unsigned long long* __restrict__ ckey,
                                            float4* __restrict__ cpos, int* __restrict__ orig) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const unsigned pv = local_pos[i];
  if (!(pv >> 31)) return;
  const unsigned d = (pv & 0x7fffffffu) + block_off[i / SCAN_BS];
  ckey[d] = skey[i];
  cpos[d] = cent[i];
  orig[d] = i;
}

// dense_seg_union_kernel with the ground edge: horizontal d2 = dx*dx + dz*dz <= tol2 and |dy| <= max_step, fp64 of
// the float centroids without FMA (y is up)
__global__ void __launch_bounds__(128)
dense_ground_union_kernel(const unsigned long long* __restrict__ skey, const float4* __restrict__ spos, int n,
                          int radius, double tol2, double max_step, int* par) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float4 pi = spos[i];
  const double px = (double)pi.x, py = (double)pi.y, pz = (double)pi.z;
  dense_box_walk(skey, n, skey[i], radius, [&](int j) {
    if (j <= i) return;
    const float4 pj = spos[j];
    const double dx = px - (double)pj.x, dy = py - (double)pj.y, dz = pz - (double)pj.z;
    if (dx * dx + dz * dz <= tol2 && fabs(dy) <= max_step) dense_seg_unite(par, i, j);
  });
}

// one thread per target voxel e: its label from the compacted labels clab (-1 when it was not selected), with
// `ground` its ground flag (label >= 0); the first *kept records' `first` from compacted position to target index
__global__ void dense_ground_scatter_kernel(int n, const unsigned* __restrict__ local_pos,
                                            const unsigned* __restrict__ block_off, const int* __restrict__ clab,
                                            const int* __restrict__ orig, const int* __restrict__ kept,
                                            loam_b200_segment* __restrict__ seg, int* __restrict__ labels,
                                            unsigned char* __restrict__ ground) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n) return;
  const unsigned pv = local_pos[e];
  const int lab = (pv >> 31) ? clab[(pv & 0x7fffffffu) + block_off[e / SCAN_BS]] : -1;
  labels[e] = lab;
  if (ground) ground[e] = lab >= 0 ? 1 : 0;
  if (kept && e < *kept) seg[e].first = orig[seg[e].first];
}

// One thread per point: q = associate_to_map(pose, p) and dense_match over the ground voxels; class 1 ground (a match
// with |pd| <= max_height, pd = (nx*(qx - cx) + ny*(qy - cy)) + nz*(qz - cz) in fp32), 0 not ground, 0xff (-1) for
// a point that is not finite or whose voxel lies outside the key range
__global__ void dense_ground_cloud_kernel(const unsigned long long* __restrict__ skey, const float4* __restrict__ cent,
                                          const float4* __restrict__ nrm, const unsigned char* __restrict__ ground,
                                          int m, float inv, int radius, float gate, const float4* __restrict__ pts,
                                          int n, MapIterArgs a, float max_height, unsigned char* __restrict__ cls) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float4 po = pts[i];
  unsigned char l = 0xff;
  if (isfinite(po.x) && isfinite(po.y) && isfinite(po.z)) {
    float qx, qy, qz;
    associate_to_map(a, po, qx, qy, qz);
    const unsigned long long key = dense_key_of(make_float4(qx, qy, qz, 0.f), inv);
    if (key != DENSE_EMPTY) {
      const int best = dense_match(skey, cent, m, key, radius, gate, qx, qy, qz, [&](int j) { return ground[j] != 0; });
      l = 0;
      if (best >= 0) {
        const float4 c = cent[best], nv = nrm[best];
        const float pd = (nv.x * (qx - c.x) + nv.y * (qy - c.y)) + nv.z * (qz - c.z);
        if (fabsf(pd) <= max_height) l = 1;
      }
    }
  }
  cls[i] = l;
}

// Scratch of one segmentation: DenseTarget::seg for the target, loam_b200_ctx::seg for clouds; kept for the next call
struct DenseSegScratch {
  DevBuf<unsigned long long> keys64, skey;  // cloud: input keys, sorted keys
  DevBuf<float4> pts, spos;                 // cloud: input points (host upload), sorted positions
  DevBuf<int> orig, inv;                    // cloud: sorted position <-> input index
  DevBuf<int> par, root, size, first, segid, segroot, start, labels, ints;
  DevBuf<double4> csum;
  DevBuf<float4> clo, chi;
  DevBuf<loam_b200_segment> out;

  void release() {
    keys64.release(); skey.release(); pts.release(); spos.release(); orig.release(); inv.release(); par.release();
    root.release(); size.release(); first.release(); segid.release(); segroot.release(); start.release();
    labels.release(); ints.release(); csum.release(); clo.release(); chi.release(); out.release();
  }
};

// Host-side state of the map (loam_b200_ctx::dense).  The insertion runs on its own stream with its own sort scratch,
// so the next sweep's stages on the main stream and the map update on its lanes neither wait for it nor share buffers.
struct DenseMap {
  float leaf = 0.f;
  unsigned long long max_voxels = 0;
  cudaStream_t stream = nullptr;
  cudaEvent_t ev_in = nullptr;    // the cloud is complete (main stream)
  cudaEvent_t ev_done = nullptr;  // the last insertion has read its cloud (and mirrored the counters to ctr_host)
  cudaEvent_t ev_observed = nullptr;  // the last visibility pass has read its cloud (never ev_done: the insertion sizes
                                      // the table from the counters only when ev_done says they are current)
  unsigned pending_slots = 0;     // cloud slots an insertion may still read: the next write waits for ev_done
  SortScratch sort;
  DevBuf<unsigned long long> keys64, skeys;
  DevBuf<unsigned> pos, rank;
  DevBuf<unsigned long long> run_key;
  DevBuf<unsigned> run_count;
  DevBuf<double4> run_sum;
  DevBuf<long long> run_slot;
  DevBuf<int> slots, ints;        // export: slot of each compacted voxel; [0] runs, [1] new voxels, [2] compaction counter
  DevBuf<float4> out;
  DevBuf<unsigned> out_count, out_evidence;
  DevBuf<float4> normals;         // export with normals: (nx, ny, nz, curvature) per exported voxel
  DevBuf<double4> xsum;           // snapshot / merge: the entries' sums, counts and packed evidence (merge: in input
  DevBuf<unsigned> xcount, xev;   // order, the sums transformed in place), and the evidence of the merge's runs
  DevBuf<unsigned> run_ev;
  double vis_h_res = 0.0, vis_v_res = 0.0, vis_margin = 0.0;  // visibility pass (vis_h_res == 0: off)
  int vis_rows = 0, vis_cols = 0;
  DevBuf<unsigned> image;         // range image of the sweep being observed (float bits, DENSE_NO_RETURN when empty)
  double carve_margin = 0.0, carve_max = 0.0;  // carve mode (carve_max == 0: off)
  DenseBrickIndex live;                        // carve mode's occupancy index (stream-ordered allocations on `stream`;
                                               // no slots: carve mode off, or dropped by a clear)
  unsigned long long live_bound = 0;           // upper bound of its bricks, known without a readback
  unsigned* stamp = nullptr;                   // carve mode's per-slot stamps (table_size words once allocated)
  unsigned long long stamp_size = 0;
  unsigned epoch = 0;                          // the last carve pass (stamps 2e / 2e + 1)
  DevBuf<DenseCounters> ctr;
  PinBuf<DenseCounters> ctr_host;
  DenseSlot* table = nullptr;     // stream-ordered allocation (cudaMallocAsync on `stream`)
  unsigned long long table_size = 0;
  unsigned long long bound = 0;   // upper bound of the voxels in the table, known without a readback

  // stream, events and buffers (the map's own; the context's stream must not be inside a DenseScope)
  void release() {
    if (stream) {
      cudaStreamSynchronize(stream);
      if (table) cudaFreeAsync(table, stream);
      if (live.key) cudaFreeAsync(live.key, stream);
      if (live.mask) cudaFreeAsync(live.mask, stream);
      if (stamp) cudaFreeAsync(stamp, stream);
      cudaStreamSynchronize(stream);
      cudaStreamDestroy(stream);
    }
    stream = nullptr;
    table = nullptr;
    table_size = 0;
    live = DenseBrickIndex{};
    live_bound = 0;
    stamp = nullptr;
    stamp_size = 0;
    sort.keys_a.release(); sort.keys_b.release(); sort.vals_a.release(); sort.vals_b.release(); sort.hist.release();
    keys64.release(); skeys.release(); pos.release(); rank.release(); run_key.release(); run_count.release();
    run_sum.release(); run_slot.release(); slots.release(); ints.release(); out.release(); out_count.release();
    out_evidence.release(); normals.release(); image.release();
    xsum.release(); xcount.release(); xev.release(); run_ev.release();
    ctr.release(); ctr_host.release();
    if (ev_in) cudaEventDestroy(ev_in);
    if (ev_done) cudaEventDestroy(ev_done);
    if (ev_observed) cudaEventDestroy(ev_observed);
    ev_in = ev_done = ev_observed = nullptr;
  }
};

// Registration target of loam_b200_dense_align (loam_b200_ctx::target): a snapshot of sorted keys, centroids and
// normals, built from the map's export or loaded from the host.  Independent of DenseMap, so a context without the map
// can load one.  The iteration's scratch lives beside it and is used on the context's own stream.
struct DenseTarget {
  bool ready = false;             // false until a build or load succeeds (a failed one leaves no target)
  float leaf = 0.f;
  int n = 0;
  DevBuf<unsigned long long> keys, keys64;  // sorted keys; load: the entries' keys in input order
  DevBuf<float4> cent, nrm;
  DevBuf<float4> pts;             // the cloud being aligned (a host cloud is uploaded here)
  DevBuf<MapIterArgs> args;       // the poses of one launch's hypothesis list
  DevBuf<float> partials, result; // per hypothesis: per-CTA partial sums, the folded sums (32, or 2 for a score)
  DevBuf<unsigned> ticket;        // per hypothesis; zero between launches (the reductions reset it)
  DevBuf<int> match, flag;
  DevBuf<float4> coeff;
  DevBuf<int8_t> sel;
  // ray index of loam_b200_dense_raycast: built on the first cast after a build or load (slots once built).  Its
  // pointers alias the ray_* buffers below, so those are reserved only by dense_ray_index_build, which runs only while
  // `ray` is empty (a build, load or release empties it first).
  DenseBrickIndex ray;
  DevBuf<unsigned long long> ray_key, ray_mask;
  DevBuf<unsigned> ray_base;
  DevBuf<int> ray_idx;
  DevBuf<float> ray_range;        // the cast's outputs
  DevBuf<int> ray_hit;
  // place database of loam_b200_dense_place_build: place_k descriptors of the params' cells (place_k == 0: none; a
  // build, load or release drops it), the candidates' positions kept on the host for the global relocalisation
  int place_k = 0;
  DensePlaceArgs place_args{};
  std::vector<float> place_pos;
  DevBuf<unsigned> place_db, place_q;   // database; the query's descriptor
  DevBuf<float> place_posd;             // positions during a build
  DevBuf<double2> place_tab;            // sector boundaries of the call's params
  DevBuf<double> place_dist;            // per candidate: best distance and shift of the last query
  DevBuf<int> place_shift;
  // distance field of loam_b200_dense_distance_build: the box's sq field (dist_ready false: none; a build, load or
  // release drops it), the EDT's scratch (kept for the next build) and the query's outputs
  bool dist_ready = false;
  DenseDistArgs dist_args{};
  DevBuf<int> dist_sq;
  DevBuf<float> dist_f;                 // the float distances of a build that downloads them
  DevBuf<int> edt_g, edt_b, edt_s, edt_t, edt_v;
  DevBuf<float> qdist, qgrad;
  DenseSegScratch seg;                  // loam_b200_dense_segment (and the ground calls' compacted entries)
  // ground of loam_b200_dense_ground: one flag per voxel in key order (ground_ready false: none; a build, load or
  // release drops it, the next dense_ground replaces it); the scratch of the ground calls
  bool ground_ready = false;
  DevBuf<unsigned char> ground, gcls;   // flags; classes of the compaction (target voxels, or a cloud's points)
  DevBuf<unsigned> gpos, gbsum;         // compact_count_kernel's local positions and block sums
  DevBuf<int> glabels;                  // labels in target order
  DevBuf<float4> gout;                  // ground_cloud: the points that are not ground, for a host copy

  void release() {
    keys.release(); keys64.release(); cent.release(); nrm.release(); pts.release(); args.release(); partials.release();
    result.release(); ticket.release(); match.release(); flag.release(); coeff.release(); sel.release();
    ray_key.release(); ray_mask.release(); ray_base.release(); ray_idx.release(); ray_range.release();
    ray_hit.release();
    place_db.release(); place_q.release(); place_posd.release(); place_tab.release(); place_dist.release();
    place_shift.release();
    place_pos.clear();
    place_k = 0;
    dist_sq.release(); dist_f.release(); edt_g.release(); edt_b.release(); edt_s.release(); edt_t.release();
    edt_v.release(); qdist.release(); qgrad.release();
    seg.release();
    ground.release(); gcls.release(); gpos.release(); gbsum.release(); glabels.release(); gout.release();
    ground_ready = false;
    dist_ready = false;
    ray = DenseBrickIndex{};
    n = 0;
    ready = false;
  }
};

}  // namespace loamb
