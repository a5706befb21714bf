// Scan-registration kernels: one CTA per scan ring does everything BasicScanRegistration::extractFeatures does
// for that ring (BasicScanRegistration.cpp:155-254):
//   setScanBuffersFor   (:321-363)  unreliable-point mask
//   setRegionBuffersFor (:284-318)  curvature + stable ascending order per feature region
//   corner / flat pick with markAsPicked neighbour suppression (:197-235, :367-386)
//   less-flat collection (:238-242) and the per-ring 0.2 m VoxelGrid (:246-252)
// The ring (<= 4096 points) lives in shared memory after one coalesced float4 pass over the ring-ordered sweep
// buffer; all arithmetic reproduces the reference's fp32 operation order (no FMA, double-promoted literals).
#pragma once

#include "ctx.cuh"

namespace loamb {

constexpr int FEAT_THREADS = 512;
constexpr int LABEL_OUTSIDE = 127;

struct FeatParams {
  int nFeatureRegions, curvatureRegion, maxCornerSharp, maxCornerLessSharp, maxSurfaceFlat;
  float lessFlatFilterSize, surfaceCurvatureThreshold;
  int cap_sharp, cap_less, cap_flat;  // per-ring slot sizes
};

__device__ __forceinline__ float sqdiff(const float4& a, const float4& b) {
  // calcSquaredDiff (math_utils.h:68-76)
  const float dx = a.x - b.x, dy = a.y - b.y, dz = a.z - b.z;
  return dx * dx + dy * dy + dz * dz;
}
__device__ __forceinline__ float sqdiff_w(const float4& a, const float4& b, float wb) {
  // calcSquaredDiff with weight on the second point (math_utils.h:87-95)
  const float dx = a.x - b.x * wb, dy = a.y - b.y * wb, dz = a.z - b.z * wb;
  return dx * dx + dy * dy + dz * dz;
}
__device__ __forceinline__ float sqnorm(const float4& p) { return p.x * p.x + p.y * p.y + p.z * p.z; }

// markAsPicked (:367-386) executed by one warp: lane 0 marks the point, lanes 1..cr test the forward gaps,
// lanes 17..16+cr the backward gaps; the first gap (ballot + ffs) bounds the marked extent.
__device__ __forceinline__ void mark_as_picked_warp(const float4* P, int8_t* picked, int li, int cr, int lane) {
  bool fgap = false, bgap = false;
  if (lane >= 1 && lane <= cr) fgap = (double)sqdiff(P[li + lane], P[li + lane - 1]) > 0.05;
  const int bl = lane - 16;
  if (bl >= 1 && bl <= cr) bgap = (double)sqdiff(P[li - bl], P[li - bl + 1]) > 0.05;
  const unsigned fm = __ballot_sync(0xffffffffu, fgap);
  const unsigned bm = __ballot_sync(0xffffffffu, bgap) >> 16;
  const int fext = fm ? (__ffs(fm) - 1) - 1 : cr;  // lanes are 1-based: first gap at lane g -> extent g-1
  const int bext = bm ? (__ffs(bm) - 1) - 1 : cr;
  __syncwarp();  // every lane's read of picked[] for this pick (the caller's eligibility test) precedes the marks
  if (lane == 0) picked[li] = 1;
  if (lane >= 1 && lane <= fext) picked[li + lane] = 1;
  if (bl >= 1 && bl <= bext) picked[li - bl] = 1;
  __syncwarp();
}

// shared-memory bitonic sort of 64-bit keys (n2 = power of two); one thread per compare-exchange PAIR
__device__ __forceinline__ void bitonic_sort_u64(unsigned long long* a, int n2) {
  const int half = n2 >> 1;
  for (int k = 2; k <= n2; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int p = threadIdx.x; p < half; p += blockDim.x) {
        const int t = ((p & ~(j - 1)) << 1) | (p & (j - 1));  // lower element of pair p at distance j
        const int ixj = t | j;
        const unsigned long long x = a[t], y = a[ixj];
        const bool up = ((t & k) == 0);
        if ((x > y) == up) { a[t] = y; a[ixj] = x; }
      }
      __syncthreads();
    }
  }
}

// Dynamic shared memory layout for a ring of n points (n rounded up to ncap):
//   float4 P[ncap] | float curv[ncap] | int order[ncap] | u64 vkeys[n2] | int8 picked[ncap] | int8 label[ncap]
__global__ void __launch_bounds__(FEAT_THREADS, 1)
feature_ring_kernel(const float4* __restrict__ pts, const int* __restrict__ ring_start,
                    const int* __restrict__ ring_end, FeatParams prm, int ncap, int n2cap,
                    int* __restrict__ picks, int* __restrict__ counts, int8_t* __restrict__ label_out,
                    float4* __restrict__ lessflat_out) {
  extern __shared__ __align__(16) unsigned char smem[];
  float4* P = reinterpret_cast<float4*>(smem);
  float* curv = reinterpret_cast<float*>(P + ncap);
  int* order = reinterpret_cast<int*>(curv + ncap);
  unsigned long long* vkeys = reinterpret_cast<unsigned long long*>(order + ncap);
  int8_t* picked = reinterpret_cast<int8_t*>(vkeys + n2cap);
  int8_t* label = picked + ncap;
  __shared__ int s_scan[FEAT_THREADS / 32];
  __shared__ float s_red[6][FEAT_THREADS / 32];
  __shared__ int s_misc[8];

  const int ring = blockIdx.x;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const long long s = ring_start[ring], e = ring_end[ring];
  const int cr = prm.curvatureRegion;
  const int slots = prm.cap_sharp + prm.cap_less + prm.cap_flat;
  int* my_picks = picks + (size_t)ring * slots;

  // "skip empty scans" (:165): size_t compare, e may be s-1 for an empty ring (then e <= s + 2cr holds as well)
  if (e <= s + 2 * cr) {
    if (tid < 4) counts[ring * 4 + tid] = 0;
    if (label_out)
      for (long long i = s + tid; i <= e; i += blockDim.x) label_out[i] = LABEL_OUTSIDE;
    return;
  }
  const int n = (int)(e - s + 1);

  for (int i = tid; i < n; i += blockDim.x) {
    P[i] = pts[s + i];
    picked[i] = 0;
    label[i] = LABEL_OUTSIDE;
  }
  __syncthreads();

  // ---- unreliable points (:328-362).  Iterations only read points and OR marks, so they run in parallel; the
  // `continue` at :345 only skips the second test of the same i.
  for (int i = cr + tid; i < n - 1 - cr; i += blockDim.x) {
    const float4 prev = P[i - 1], cur = P[i], nxt = P[i + 1];
    const float diffNext = sqdiff(nxt, cur);
    bool skip = false;
    if ((double)diffNext > 0.1) {
      const float depth1 = sqrtf(sqnorm(cur));
      const float depth2 = sqrtf(sqnorm(nxt));
      if (depth1 > depth2) {
        const float wd = sqrtf(sqdiff_w(nxt, cur, depth2 / depth1)) / depth2;
        if ((double)wd < 0.1) {
          for (int k = 0; k <= cr; k++) picked[i - cr + k] = 1;
          skip = true;
        }
      } else {
        const float wd = sqrtf(sqdiff_w(cur, nxt, depth1 / depth2)) / depth1;
        if ((double)wd < 0.1)
          for (int k = 0; k <= cr; k++) picked[i + 1 + k] = 1;
      }
    }
    if (!skip) {
      const float diffPrev = sqdiff(cur, prev);
      const float dis = sqnorm(cur);
      if ((double)diffNext > 0.0002 * (double)dis && (double)diffPrev > 0.0002 * (double)dis) picked[i] = 1;
    }
  }

  // ---- curvature for every point of every region (:293-308); regions tile [cr, n-2-cr] contiguously
  const float w = (float)(-2 * cr);
  for (int i = cr + tid; i <= n - 2 - cr; i += blockDim.x) {
    float dx = w * P[i].x, dy = w * P[i].y, dz = w * P[i].z;
    for (int j = 1; j <= cr; j++) {
      dx += P[i + j].x + P[i - j].x;
      dy += P[i + j].y + P[i - j].y;
      dz += P[i + j].z + P[i - j].z;
    }
    curv[i] = dx * dx + dy * dy + dz * dz;
  }
  __syncthreads();

  // ---- region bounds (:180-183), all in unsigned 64-bit like the reference's size_t
  const int nreg = prm.nFeatureRegions;
  // ---- stable ascending order of the points of every region (:311-317 is a stable insertion sort): ONE bitonic sort
  // of (region, curvature bits, index) keys over the whole ring -- curvatures are sums of squares (>= +0), so their bit
  // patterns order like the floats; the index breaks ties the way a stable sort does.  (The first version ranked every
  // point against its whole region, O(n^2), and that ranking dominated the kernel's instructions.)
  int n2r = 1;
  while (n2r < n) n2r <<= 1;
  for (int t = tid; t < n2r; t += blockDim.x) vkeys[t] = ~0ull;
  __syncthreads();
  for (int j = 0; j < nreg; j++) {
    const unsigned long long a = (unsigned long long)(s + cr), b = (unsigned long long)(e - cr);
    const unsigned long long sp = (a * (unsigned long long)(nreg - j) + b * (unsigned long long)j) / (unsigned long long)nreg;
    const unsigned long long ep = (a * (unsigned long long)(nreg - 1 - j) + b * (unsigned long long)(j + 1)) / (unsigned long long)nreg - 1ull;
    if (ep <= sp) continue;
    const int lsp = (int)(sp - (unsigned long long)s), lep = (int)(ep - (unsigned long long)s);
    for (int i = lsp + tid; i <= lep; i += blockDim.x) {
      vkeys[i] = ((unsigned long long)j << 52) | ((unsigned long long)__float_as_uint(curv[i]) << 20) | (unsigned long long)i;
      label[i] = 0;  // SURFACE_LESS_FLAT (:290)
    }
  }
  __syncthreads();
  bitonic_sort_u64(vkeys, n2r);
  // sorted position p of the ring <-> point index vkeys[p] & 0xfffff; region j's points follow those of regions < j

  // ---- greedy picks, sequential over regions, executed by warp 0 (:197-235)
  if (warp == 0) {
    int n_sharp = 0, n_less = 0, n_flat = 0;
    int roff = 0;  // sorted position of the current region's first point
    const float thr = prm.surfaceCurvatureThreshold;
    for (int j = 0; j < nreg; j++) {
      const unsigned long long a = (unsigned long long)(s + cr), b = (unsigned long long)(e - cr);
      const unsigned long long sp = (a * (unsigned long long)(nreg - j) + b * (unsigned long long)j) / (unsigned long long)nreg;
      const unsigned long long ep = (a * (unsigned long long)(nreg - 1 - j) + b * (unsigned long long)(j + 1)) / (unsigned long long)nreg - 1ull;
      if (ep <= sp) continue;
      const int lsp = (int)(sp - (unsigned long long)s), lep = (int)(ep - (unsigned long long)s);
      const int nr = lep - lsp + 1;

      // corners: descending curvature
      int largest = 0;
      for (int k = nr; k > 0 && largest < prm.maxCornerLessSharp; k -= 32) {
        const int pos = k - 1 - lane;
        const int idx = pos >= 0 ? (int)(vkeys[roff + pos] & 0xfffffull) : -1;
        const bool above = idx >= 0 && curv[idx] > thr;
        const unsigned m_above = __ballot_sync(0xffffffffu, above);
        if (m_above == 0u) break;
        int done_upto = -1;
        while (largest < prm.maxCornerLessSharp) {
          const bool elig = above && lane > done_upto && picked[idx] == 0;
          const unsigned m = __ballot_sync(0xffffffffu, elig);
          if (m == 0u) break;
          const int l = __ffs(m) - 1;
          const int pidx = __shfl_sync(0xffffffffu, idx, l);
          largest++;
          if (lane == 0) {
            if (largest <= prm.maxCornerSharp) {
              label[pidx] = 2;  // CORNER_SHARP
              my_picks[n_sharp] = (int)s + pidx;
            } else {
              label[pidx] = 1;  // CORNER_LESS_SHARP
            }
            my_picks[prm.cap_sharp + n_less] = (int)s + pidx;
          }
          if (largest <= prm.maxCornerSharp) n_sharp++;
          n_less++;
          mark_as_picked_warp(P, picked, pidx, cr, lane);
          done_upto = l;
        }
        if (m_above != 0xffffffffu) break;  // sorted: everything further down is below the threshold too
      }

      // flats: ascending curvature
      int smallest = 0;
      for (int k = 0; k < nr && smallest < prm.maxSurfaceFlat; k += 32) {
        const int pos = k + lane;
        const int idx = pos < nr ? (int)(vkeys[roff + pos] & 0xfffffull) : -1;
        const bool below = idx >= 0 && curv[idx] < thr;
        const unsigned m_below = __ballot_sync(0xffffffffu, below);
        if (m_below == 0u) break;
        int done_upto = -1;
        while (smallest < prm.maxSurfaceFlat) {
          const bool elig = below && lane > done_upto && picked[idx] == 0;
          const unsigned m = __ballot_sync(0xffffffffu, elig);
          if (m == 0u) break;
          const int l = __ffs(m) - 1;
          const int pidx = __shfl_sync(0xffffffffu, idx, l);
          smallest++;
          if (lane == 0) {
            label[pidx] = -1;  // SURFACE_FLAT
            my_picks[prm.cap_sharp + prm.cap_less + n_flat] = (int)s + pidx;
          }
          n_flat++;
          mark_as_picked_warp(P, picked, pidx, cr, lane);
          done_upto = l;
        }
        if (m_below != 0xffffffffu) break;
      }
      roff += nr;
    }
    if (lane == 0) {
      counts[ring * 4 + 0] = n_sharp;
      counts[ring * 4 + 1] = n_less;
      counts[ring * 4 + 2] = n_flat;
    }
  }
  __syncthreads();

  if (label_out)
    for (int i = tid; i < n; i += blockDim.x) label_out[s + i] = label[i];

  // ---- less-flat collection (:238-242): order-preserving compaction of label <= 0 (regions ascend contiguously)
  // chunked block scan; positions stored in `order` (no longer needed)
  int base = 0;
  for (int c0 = 0; c0 < n; c0 += blockDim.x) {
    const int i = c0 + tid;
    const bool f = i < n && label[i] <= 0;
    const unsigned bm = __ballot_sync(0xffffffffu, f);
    if (lane == 0) s_scan[warp] = __popc(bm);
    __syncthreads();
    int woff = 0, tot = 0;
    for (int wv = 0; wv < FEAT_THREADS / 32; wv++) {
      if (wv < warp) woff += s_scan[wv];
      tot += s_scan[wv];
    }
    if (f) order[base + woff + __popc(bm & ((1u << lane) - 1u))] = i;
    base += tot;
    __syncthreads();
  }
  const int nlf = base;
  if (nlf == 0) {
    if (tid == 0) counts[ring * 4 + 3] = 0;
    return;
  }

  // ---- per-ring VoxelGrid (pcl::VoxelGrid semantics: bbox -> integer voxel index -> sort -> centroid per run)
  float mn[3] = {FLT_MAX, FLT_MAX, FLT_MAX}, mx[3] = {-FLT_MAX, -FLT_MAX, -FLT_MAX};
  for (int t = tid; t < nlf; t += blockDim.x) {
    const float4 p = P[order[t]];
    mn[0] = fminf(mn[0], p.x); mx[0] = fmaxf(mx[0], p.x);
    mn[1] = fminf(mn[1], p.y); mx[1] = fmaxf(mx[1], p.y);
    mn[2] = fminf(mn[2], p.z); mx[2] = fmaxf(mx[2], p.z);
  }
  for (int a = 0; a < 3; a++) {
    for (int o = 16; o > 0; o >>= 1) {
      mn[a] = fminf(mn[a], __shfl_xor_sync(0xffffffffu, mn[a], o));
      mx[a] = fmaxf(mx[a], __shfl_xor_sync(0xffffffffu, mx[a], o));
    }
    if (lane == 0) { s_red[a][warp] = mn[a]; s_red[3 + a][warp] = mx[a]; }
  }
  __syncthreads();
  for (int a = 0; a < 3; a++) {
    float vmn = FLT_MAX, vmx = -FLT_MAX;
    for (int wv = 0; wv < FEAT_THREADS / 32; wv++) { vmn = fminf(vmn, s_red[a][wv]); vmx = fmaxf(vmx, s_red[3 + a][wv]); }
    mn[a] = vmn; mx[a] = vmx;
  }
  const float leaf = prm.lessFlatFilterSize;
  const float inv = 1.0f / leaf;
  const long long dxv = (long long)((mx[0] - mn[0]) * inv) + 1, dyv = (long long)((mx[1] - mn[1]) * inv) + 1,
                  dzv = (long long)((mx[2] - mn[2]) * inv) + 1;
  float4* out = lessflat_out + s;  // ring slot (capacity n)
  if (dxv * dyv * dzv > 2147483647ll) {
    // "leaf size too small": pcl returns the input unchanged
    for (int t = tid; t < nlf; t += blockDim.x) out[t] = P[order[t]];
    if (tid == 0) counts[ring * 4 + 3] = nlf;
    return;
  }
  const int minb0 = (int)floorf(mn[0] * inv), minb1 = (int)floorf(mn[1] * inv), minb2 = (int)floorf(mn[2] * inv);
  const int div0 = (int)floorf(mx[0] * inv) - minb0 + 1, div1 = (int)floorf(mx[1] * inv) - minb1 + 1;
  int n2 = 1;
  while (n2 < nlf) n2 <<= 1;
  for (int t = tid; t < n2; t += blockDim.x) {
    unsigned long long key = ~0ull;
    if (t < nlf) {
      const float4 p = P[order[t]];
      const int i0 = (int)(floorf(p.x * inv) - (float)minb0);
      const int i1 = (int)(floorf(p.y * inv) - (float)minb1);
      const int i2 = (int)(floorf(p.z * inv) - (float)minb2);
      // unsigned: pcl's int32 key wraps (defined behaviour here) when the div product passes 2^31
      const unsigned vidx = (unsigned)i0 + (unsigned)i1 * (unsigned)div0 + (unsigned)i2 * (unsigned)div0 * (unsigned)div1;
      key = ((unsigned long long)vidx << 32) | (unsigned)t;
    }
    vkeys[t] = key;
  }
  __syncthreads();
  bitonic_sort_u64(vkeys, n2);

  // run heads -> output slot via chunked scan; each head averages its run in sorted order
  base = 0;
  for (int c0 = 0; c0 < nlf; c0 += blockDim.x) {
    const int t = c0 + tid;
    const bool head = t < nlf && (t == 0 || (unsigned)(vkeys[t] >> 32) != (unsigned)(vkeys[t - 1] >> 32));
    const unsigned bm = __ballot_sync(0xffffffffu, head);
    if (lane == 0) s_scan[warp] = __popc(bm);
    __syncthreads();
    int woff = 0, tot = 0;
    for (int wv = 0; wv < FEAT_THREADS / 32; wv++) {
      if (wv < warp) woff += s_scan[wv];
      tot += s_scan[wv];
    }
    if (head) {
      const unsigned v = (unsigned)(vkeys[t] >> 32);
      float sx = 0.f, sy = 0.f, sz = 0.f, si = 0.f;
      int cnt = 0;
      for (int u = t; u < nlf && (unsigned)(vkeys[u] >> 32) == v; u++) {
        const float4 p = P[order[(unsigned)(vkeys[u] & 0xffffffffu)]];
        sx += p.x; sy += p.y; sz += p.z; si += p.w;
        cnt++;
      }
      const float fn = (float)cnt;
      out[base + woff + __popc(bm & ((1u << lane) - 1u))] = make_float4(sx / fn, sy / fn, sz / fn, si / fn);
    }
    base += tot;
    __syncthreads();
  }
  if (tid == 0) counts[ring * 4 + 3] = base;
  (void)s_misc;
}

// pack per-ring results densely, one CTA per ring: three pick lists (indices + gathered points) and the less-flat DS
// cloud, ring-major.  Offsets are exclusive sums of the per-ring counts (R <= 256, one block-wide reduction each).
__global__ void __launch_bounds__(256)
feature_pack_kernel(const int* __restrict__ counts, const int* __restrict__ picks, const int* __restrict__ ring_start,
                    const float4* __restrict__ pts, const float4* __restrict__ lessflat_slots, int n_rings,
                    FeatParams prm, int* __restrict__ sharp, int* __restrict__ less, int* __restrict__ flat,
                    float4* __restrict__ sharp_pts, float4* __restrict__ less_pts, float4* __restrict__ flat_pts,
                    float4* __restrict__ lessflat, int* __restrict__ totals) {
  __shared__ int s_off[4], s_tot[4];
  __shared__ int s_w[8][8];
  const int r = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  int before[4] = {0, 0, 0, 0}, all[4] = {0, 0, 0, 0};
  if (tid < n_rings) {
#pragma unroll
    for (int k = 0; k < 4; k++) {
      const int c = counts[tid * 4 + k];
      all[k] = c;
      before[k] = tid < r ? c : 0;
    }
  }
#pragma unroll
  for (int k = 0; k < 4; k++) {
    int b = before[k], a = all[k];
    for (int o = 16; o > 0; o >>= 1) {
      b += __shfl_xor_sync(0xffffffffu, b, o);
      a += __shfl_xor_sync(0xffffffffu, a, o);
    }
    if (lane == 0) { s_w[warp][k] = b; s_w[warp][4 + k] = a; }
  }
  __syncthreads();
  if (tid < 4) {
    int b = 0, a = 0;
    for (int w = 0; w < 8; w++) { b += s_w[w][tid]; a += s_w[w][4 + tid]; }
    s_off[tid] = b;
    s_tot[tid] = a;
    if (r == 0) totals[tid] = a;
  }
  __syncthreads();
  const int slots = prm.cap_sharp + prm.cap_less + prm.cap_flat;
  const int* pk = picks + (size_t)r * slots;
  const int ns = counts[r * 4 + 0], nl = counts[r * 4 + 1], nf = counts[r * 4 + 2], nd = counts[r * 4 + 3];
  for (int i = tid; i < ns; i += blockDim.x) { const int ix = pk[i]; sharp[s_off[0] + i] = ix; sharp_pts[s_off[0] + i] = pts[ix]; }
  for (int i = tid; i < nl; i += blockDim.x) { const int ix = pk[prm.cap_sharp + i]; less[s_off[1] + i] = ix; less_pts[s_off[1] + i] = pts[ix]; }
  for (int i = tid; i < nf; i += blockDim.x) { const int ix = pk[prm.cap_sharp + prm.cap_less + i]; flat[s_off[2] + i] = ix; flat_pts[s_off[2] + i] = pts[ix]; }
  const float4* src = lessflat_slots + ring_start[r];
  for (int i = tid; i < nd; i += blockDim.x) lessflat[s_off[3] + i] = src[i];
}

}  // namespace loamb
