// Fused scan-to-map Gauss-Newton iteration (SURVEY.md §8a M1-M5).
// Eight lanes per stack point: pointAssociateToMap (BasicLaserMapping.cpp:207-219) -> exact 5-NN against the corner /
// surface map through the 1 m uniform grid of gridnn.cuh, the d5^2 < 1.0 gate (:669-671, :758-760) being what makes
// the fixed-radius search exact -> PCA line fit (:673-710) or
// 5x3 least-squares plane fit (:762-791) -> residual weight (:712-749, :795-814) -> Jacobian row (:842-861) ->
// warp-shuffle tree reduction of the 21 + 6 normal-equation accumulators (+ counts), one partial per CTA,
// combined in fixed order by the last CTA to finish (deterministic run to run).
#pragma once

#include "gridnn.cuh"
#include "lbvh.cuh"
#include "linalg.cuh"
#include "lmstep.cuh"
#include "lmstep_warp.cuh"

namespace loamb {

constexpr int LM_THREADS = 128;
constexpr int NEQ = 32;  // 21 AtA (upper triangle, row-major) + 6 AtB + n_selected + n_corner_selected + 3 pad

struct MapIterArgs {
  float srx, crx, sry, cry, srz, crz;  // sin / cos of rot_x, rot_y, rot_z as cached by the host's Angle objects
  float tx, ty, tz;
  float A[9], B[9], C[9];              // Jacobian coefficient matrices, products formed on the host in reference order
};

// sin / cos of the pose angles -> kernel arguments (BasicLaserMapping.cpp:842-853), host and device
LOAMB_HD inline void map_args_from(const float sin_[3], const float cos_[3], const float pos[3], MapIterArgs& a) {
  const float srx = sin_[0], crx = cos_[0], sry = sin_[1], cry = cos_[1], srz = sin_[2],
              crz = cos_[2];
  a.srx = srx; a.crx = crx; a.sry = sry; a.cry = cry; a.srz = srz; a.crz = crz;
  a.tx = pos[0]; a.ty = pos[1]; a.tz = pos[2];
  // Jacobian coefficient products, formed left to right exactly like BasicLaserMapping.cpp:842-853
  a.A[0] = crx * sry * srz;      a.A[1] = crx * crz * sry;        a.A[2] = -(srx * sry);
  a.A[3] = -srx * srz;           a.A[4] = -(crz * srx);           a.A[5] = -crx;
  a.A[6] = crx * cry * srz;      a.A[7] = crx * cry * crz;        a.A[8] = -(cry * srx);
  a.B[0] = cry * srx * srz - crz * sry;
  a.B[1] = sry * srz + cry * crz * srx;
  a.B[2] = crx * cry;
  a.B[3] = a.B[4] = a.B[5] = 0.f;
  a.B[6] = -cry * crz - srx * sry * srz;
  a.B[7] = cry * srz - crz * srx * sry;
  a.B[8] = -(crx * sry);
  a.C[0] = crz * srx * sry - cry * srz;
  a.C[1] = -cry * crz - srx * sry * srz;
  a.C[2] = 0.f;
  a.C[3] = crx * crz;
  a.C[4] = -(crx * srz);
  a.C[5] = 0.f;
  a.C[6] = sry * srz + cry * crz * srx;
  a.C[7] = crz * sry - cry * srx * srz;
  a.C[8] = 0.f;
}

// ---- device-resident Gauss-Newton loop (lmstep.cuh)
// what the iteration kernel of the device-resident loop works on (see OdomLoopIo); the two cell lookups are stored as
// raw bytes because their type depends on the search structure in use (MapCellLookup / GridCellLookup)
constexpr int MAP_LOOKUP_BYTES = 128;
struct MapLoopIo {
  alignas(16) unsigned char lookup[2][MAP_LOOKUP_BYTES];
  const float4* queries;       // corner queries
  const float4* queries_surf;  // surface queries (the two down-sized stacks are separate clouds)
  int n_corner_total, c0, n_corner, s0, n_surf, corner_blocks, n_blocks;
  int min_corner_map, min_surf_map;  // sizes of the from-map clouds (the <= 10 / <= 100 gate is evaluated by the host)
};
struct MapLmState {
  LmHeader h;
  GnState gn;
  float delta_t_abort, delta_r_abort;
  int max_iter;
  MapIterArgs args;  // arguments of iteration h.iter
  MapLoopIo io;
};

#if defined(__CUDACC__)
// first node of the loop graph: the WHILE condition for iteration 0 (a loop with nothing to do posts at once)
__global__ void lm_gate_kernel(const LmHeader* h, unsigned long long handle, float* mailbox_host) {
  if (threadIdx.x == 0 && blockIdx.x == 0) lm_loop_control(*h, handle, mailbox_host);
}

__device__ inline void map_lm_refresh_args(MapLmState* st) {
  float sn[3], cs[3];
  for (int i = 0; i < 3; i++) {
    double sd, cd;
    sincos((double)st->h.rot[i], &sd, &cd);  // rounded once: agrees with the host's float libm except in rare cases
    sn[i] = (float)sd;
    cs[i] = (float)cd;
  }
  MapIterArgs a;
  map_args_from(sn, cs, st->h.pos, a);
  st->args = a;
}

__global__ void map_lm_init_kernel(MapLmState* st, float rx, float ry, float rz, float tx, float ty, float tz,
                                   float delta_t_abort, float delta_r_abort, int max_iter, MapLoopIo io, int mb_seq) {
  if (threadIdx.x < (int)(sizeof(MapLoopIo) / 4) && blockIdx.x == 0)
    reinterpret_cast<int*>(&st->io)[threadIdx.x] = reinterpret_cast<const int*>(&io)[threadIdx.x];
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  st->h.mb_seq = mb_seq;
  st->h.rot[0] = rx; st->h.rot[1] = ry; st->h.rot[2] = rz;
  st->h.pos[0] = tx; st->h.pos[1] = ty; st->h.pos[2] = tz;
  st->h.iter = 0;
  st->h.done = max_iter <= 0 ? 1 : 0;
  st->h.iters_run = 0;
  st->gn.degenerate = 0;
  st->delta_t_abort = delta_t_abort;
  st->delta_r_abort = delta_r_abort;
  st->max_iter = max_iter;
  map_lm_refresh_args(st);
}

// One warp, after the normal equations of iteration h.iter are complete in s_r[0..31] (shared memory)
// (BasicLaserMapping.cpp:826-828 skip, :867-922 solve / update / convergence); lmstep_warp.cuh
__device__ inline void map_lm_step_warp(MapLmState* st, const float* s_r) {
  const int lane = threadIdx.x & 31;
  const int iter = st->h.iter;
  float rot[3], pos[3];
#pragma unroll
  for (int i = 0; i < 3; i++) { rot[i] = st->h.rot[i]; pos[i] = st->h.pos[i]; }
  bool converged = false;
  if ((int)(s_r[27] + 0.5f) >= 50) {
    float x[6];
    gn_solve_warp(s_r, iter == 0, 100.f, &st->gn, x);
#pragma unroll
    for (int i = 0; i < 3; i++) {
      rot[i] = rot[i] + x[i];
      pos[i] += x[3 + i];
    }
    float deltaR, deltaT;
    gn_deltas(x, deltaR, deltaT);
    converged = deltaR < st->delta_r_abort && deltaT < st->delta_t_abort;
  }
  // arguments of the next iteration: sin / cos of the three angles on lanes 0..2 (double sincos rounded once: agrees
  // with the host's float libm except in rare cases), the coefficient products on lane 0
  double sd, cd;
  sincos((double)(lane == 1 ? rot[1] : (lane == 2 ? rot[2] : rot[0])), &sd, &cd);
  const float sn = (float)sd, cs = (float)cd;
  float s3[3], c3[3];
#pragma unroll
  for (int i = 0; i < 3; i++) {
    s3[i] = __shfl_sync(0xffffffffu, sn, i);
    c3[i] = __shfl_sync(0xffffffffu, cs, i);
  }
  if (lane == 0) {
    MapIterArgs a;
    map_args_from(s3, c3, pos, a);
    st->args = a;
#pragma unroll
    for (int i = 0; i < 3; i++) { st->h.rot[i] = rot[i]; st->h.pos[i] = pos[i]; }
    st->h.iters_run = iter + 1;
    st->h.iter = iter + 1;
    if (converged || iter + 1 >= st->max_iter) st->h.done = 1;
    __threadfence();
  }
  __syncwarp();
}
#endif

__device__ __forceinline__ void associate_to_map(const MapIterArgs& a, const float4& pi, float& x, float& y, float& z) {
  // rotateZXY(po, rot_z, rot_x, rot_y) then translate (math_utils.h:196-238)
  const float x1 = a.crz * pi.x - a.srz * pi.y;
  const float y1 = a.srz * pi.x + a.crz * pi.y;
  const float y2 = a.crx * y1 - a.srx * pi.z;
  const float z2 = a.srx * y1 + a.crx * pi.z;
  const float x3 = a.cry * x1 + a.sry * z2;
  const float z3 = a.cry * z2 - a.sry * x1;
  x = x3 + a.tx;
  y = y2 + a.ty;
  z = z3 + a.tz;
}

// Jacobian row of a selected correspondence with coefficient `coeff` at sensor-frame point po, and its right-hand side
// (BasicLaserMapping.cpp:842-861); shared by the scan-to-map kernels and the whole-run map alignment (densemap.cuh)
__device__ __forceinline__ void map_jacobian_row(const MapIterArgs& a, const float4& po, const float4& coeff,
                                                 float row[6], float& rhs) {
  row[0] = (a.A[0] * po.x + a.A[1] * po.y + a.A[2] * po.z) * coeff.x +
           (a.A[3] * po.x + a.A[4] * po.y + a.A[5] * po.z) * coeff.y +
           (a.A[6] * po.x + a.A[7] * po.y + a.A[8] * po.z) * coeff.z;
  row[1] = (a.B[0] * po.x + a.B[1] * po.y + a.B[2] * po.z) * coeff.x +
           (a.B[6] * po.x + a.B[7] * po.y + a.B[8] * po.z) * coeff.z;
  row[2] = (a.C[0] * po.x + a.C[1] * po.y) * coeff.x + (a.C[3] * po.x + a.C[4] * po.y) * coeff.y +
           (a.C[6] * po.x + a.C[7] * po.y) * coeff.z;
  row[3] = coeff.x;
  row[4] = coeff.y;
  row[5] = coeff.z;
  rhs = -coeff.w;
}

// stack points: pointAssociateToMap with the predicted pose then pointAssociateTobeMapped back into the sensor frame
// (BasicLaserMapping.cpp:282-292 and :512-516; the round trip is not an identity in fp32 and is reproduced).
// Negated angles flip the sine only (Angle.h:47-53).
__device__ __forceinline__ float4 stack_roundtrip(const MapIterArgs& a, const float4& q) {
  float x, y, z;
  associate_to_map(a, q, x, y, z);
  // pointAssociateTobeMapped: subtract t, rotateYXZ(-ry, -rx, -rz)
  x -= a.tx; y -= a.ty; z -= a.tz;
  const float x1 = a.cry * x + (-a.sry) * z;
  const float z1 = a.cry * z - (-a.sry) * x;
  const float y2 = a.crx * y - (-a.srx) * z1;
  const float z2 = (-a.srx) * y + a.crx * z1;
  const float x3 = a.crz * x1 - (-a.srz) * y2;
  const float y3 = (-a.srz) * x1 + a.crz * y2;
  return make_float4(x3, y3, z2, q.w);
}

// closed-form point-to-line residual shared by mapping (:712-730) and odometry (BasicLaserOdometry.cpp:319-337)
__device__ __forceinline__ void line_residual(float x0, float y0, float z0, float x1, float y1, float z1, float x2,
                                              float y2, float z2, float& la, float& lb, float& lc, float& ld2) {
  const float m11 = (x0 - x1) * (y0 - y2) - (x0 - x2) * (y0 - y1);
  const float m12 = (x0 - x1) * (z0 - z2) - (x0 - x2) * (z0 - z1);
  const float m13 = (y0 - y1) * (z0 - z2) - (y0 - y2) * (z0 - z1);
  const float a012 = sqrtf(m11 * m11 + m12 * m12 + m13 * m13);
  const float l12 = sqrtf((x1 - x2) * (x1 - x2) + (y1 - y2) * (y1 - y2) + (z1 - z2) * (z1 - z2));
  la = ((y1 - y2) * m11 + (z1 - z2) * m12) / a012 / l12;
  lb = -((x1 - x2) * m11 - (z1 - z2) * m13) / a012 / l12;
  lc = -((x1 - x2) * m12 + (y1 - y2) * m13) / a012 / l12;
  ld2 = a012 / l12;
}

// corner correspondence (:671-751). Returns true when the point is selected; coeff = (s*la, s*lb, s*lc, s*ld2)
template <typename NN>
__device__ __forceinline__ bool corner_fit(const NN& nn, float sx, float sy, float sz, float4& coeff) {
  if (nn.idx[4] < 0) return false;  // fewer than five map points with d2 < 1.0  <=>  pointSearchSqDis[4] >= 1.0
  float vx = 0.f, vy = 0.f, vz = 0.f;
#pragma unroll
  for (int j = 0; j < 5; j++) { vx += nn.x[j]; vy += nn.y[j]; vz += nn.z[j]; }
  vx /= 5.0f; vy /= 5.0f; vz /= 5.0f;
  float m[9];
#pragma unroll
  for (int i = 0; i < 9; i++) m[i] = 0.f;
#pragma unroll
  for (int j = 0; j < 5; j++) {
    const float ax = nn.x[j] - vx, ay = nn.y[j] - vy, az = nn.z[j] - vz;
    m[0] += ax * ax;  // (0,0)
    m[1] += ax * ay;  // (1,0)
    m[2] += ax * az;  // (2,0)
    m[4] += ay * ay;  // (1,1)
    m[5] += ay * az;  // (2,1)
    m[8] += az * az;  // (2,2)
  }
  m[0] /= 5.0f; m[1] /= 5.0f; m[2] /= 5.0f; m[4] /= 5.0f; m[5] /= 5.0f; m[8] /= 5.0f;
  float ev[3], V[9];
  sym_eigen<3>(m, ev, V);
  if (!(ev[2] > 3.f * ev[1])) return false;
  // end points vc +- 0.1 * v (the 0.1 literal is double in the reference, :705-710)
  const float x1 = (float)((double)vx + 0.1 * (double)V[0 + 2 * 3]);
  const float y1 = (float)((double)vy + 0.1 * (double)V[1 + 2 * 3]);
  const float z1 = (float)((double)vz + 0.1 * (double)V[2 + 2 * 3]);
  const float x2 = (float)((double)vx - 0.1 * (double)V[0 + 2 * 3]);
  const float y2 = (float)((double)vy - 0.1 * (double)V[1 + 2 * 3]);
  const float z2 = (float)((double)vz - 0.1 * (double)V[2 + 2 * 3]);
  float la, lb, lc, ld2;
  line_residual(sx, sy, sz, x1, y1, z1, x2, y2, z2, la, lb, lc, ld2);
  const float s = 1.f - 0.9f * fabsf(ld2);
  coeff = make_float4(s * la, s * lb, s * lc, s * ld2);
  return (double)s > 0.1;
}

// surface correspondence (:760-816)
template <typename NN>
__device__ __forceinline__ bool surf_fit(const NN& nn, float sx, float sy, float sz, float4& coeff) {
  if (nn.idx[4] < 0) return false;
  float A[15], b[5], x[3];
#pragma unroll
  for (int j = 0; j < 5; j++) {
    A[j + 0 * 5] = nn.x[j];
    A[j + 1 * 5] = nn.y[j];
    A[j + 2 * 5] = nn.z[j];
    b[j] = -1.f;
  }
  colpiv_qr_solve<5, 3>(A, b, x);
  float pa = x[0], pb = x[1], pc = x[2], pd = 1.f;
  const float ps = sqrtf(pa * pa + pb * pb + pc * pc);
  pa /= ps; pb /= ps; pc /= ps; pd /= ps;
#pragma unroll
  for (int j = 0; j < 5; j++)
    if ((double)fabsf(pa * nn.x[j] + pb * nn.y[j] + pc * nn.z[j] + pd) > 0.2) return false;
  const float pd2 = pa * sx + pb * sy + pc * sz + pd;
  const float s = 1.f - 0.9f * fabsf(pd2) / sqrtf(sqrtf(sx * sx + sy * sy + sz * sz));
  coeff = make_float4(s * pa, s * pb, s * pc, s * pd2);
  return (double)s > 0.1;
}

// accumulate one Jacobian row into the 29 running sums
__device__ __forceinline__ void accumulate_row(float* acc, const float* row, float b, bool is_corner) {
  int k = 0;
#pragma unroll
  for (int i = 0; i < 6; i++)
#pragma unroll
    for (int j = i; j < 6; j++) acc[k++] += row[i] * row[j];
#pragma unroll
  for (int i = 0; i < 6; i++) acc[21 + i] += row[i] * b;
  acc[27] += 1.f;
  if (is_corner) acc[28] += 1.f;
}

// Result mailbox in mapped pinned host memory: the CTA that folds the partials also posts the 32 sums across PCIe and
// then a sequence number; the host spins on the sequence number instead of paying a memcpy + stream synchronise per
// Gauss-Newton iteration (~10 us each, 7-9 per sweep).  host[0..31] = sums, host[32] = sequence.  nullptr = not used.
struct ResultMailbox {
  float* host;
  int seq;
};
__device__ __forceinline__ void mailbox_post_value(const ResultMailbox& mb, int k, float v) {
  if (mb.host) {
    mb.host[k] = v;
    __threadfence_system();
  }
}
// call after a __syncthreads() that follows every mailbox_post_value of the block
__device__ __forceinline__ void mailbox_post_seq(const ResultMailbox& mb) {
  if (mb.host && threadIdx.x == 0) {
    __threadfence_system();
    *reinterpret_cast<volatile int*>(mb.host + 32) = mb.seq;
  }
}

// ---- fused all-reduce of the normal equations over NVLink peer memory (multi-GPU, cube-sharded map) -------------------
// Every rank owns an INBOX in its HBM that all peers have mapped (CUDA IPC): world x 2 slots of 32 words + world x 2
// flags.  The CTA that folds a rank's partials stores its 32 sums straight into slot [rank][parity] of EVERY rank's inbox
// (plain stores over NVLink), fences, raises flag [rank][parity] = seq in every inbox, waits until its own inbox holds
// seq from every rank and adds the world contributions in rank order (double) -- so every rank ends up with the same
// bits, with no host involvement and no separate collective launch.  seq comes from a device-side counter the ranks
// advance in lock step (they execute the same sequence of reductions); two slots per rank (parity = seq & 1) suffice
// because a rank can run at most one reduction ahead of the slowest peer.  A bounded spin turns a lost peer into a NaN
// result instead of a hung GPU.
constexpr int PEER_MAX = 8;
struct PeerReduce {
  float* slots[PEER_MAX];      // inbox of rank p: [world][2][32] words
  unsigned* flags[PEER_MAX];   // inbox flags of rank p: [world][2]
  unsigned* seq_counter;       // this rank's reduction counter (device memory)
  int rank, world;
};
constexpr int PEER_INBOX_WORDS = PEER_MAX * 2 * 32;

// Called by the 32 first threads of ONE CTA with their folded sum `v` (lane k = sum k); returns the all-reduced sum.
// kind 0: float sums (double accumulation in rank order); kind 1: the words are ints (exact integer sum).
template <int KIND>
__device__ __forceinline__ float peer_allreduce32(const PeerReduce& pr, float v) {
  const int lane = threadIdx.x & 31;
  const unsigned seq = *pr.seq_counter + 1u;
  const int par = (int)(seq & 1u);
  for (int p = 0; p < pr.world; p++) pr.slots[p][(pr.rank * 2 + par) * 32 + lane] = v;
  __threadfence_system();
  __syncwarp();
  if (lane < pr.world) {
    *reinterpret_cast<volatile unsigned*>(&pr.flags[lane][pr.rank * 2 + par]) = seq;
    // wait for the contribution of rank `lane` in my own inbox
    const volatile unsigned* f = reinterpret_cast<volatile unsigned*>(&pr.flags[pr.rank][lane * 2 + par]);
    const long long t0 = clock64();
    while (*f != seq) {
      __nanosleep(64);
      if (clock64() - t0 > 4000000000ll) break;  // ~2 s: give up (result becomes NaN below)
    }
  }
  __syncwarp();
  __threadfence_system();
  bool ok = true;
  for (int q = 0; q < pr.world; q++)
    ok = ok && (*reinterpret_cast<volatile unsigned*>(&pr.flags[pr.rank][q * 2 + par]) == seq);
  float out;
  if (KIND == 0) {
    double acc = 0.0;
    for (int q = 0; q < pr.world; q++)
      acc += (double)*reinterpret_cast<volatile float*>(&pr.slots[pr.rank][(q * 2 + par) * 32 + lane]);
    out = ok ? (float)acc : __int_as_float(0x7fc00000);
  } else {
    int acc = 0;
    for (int q = 0; q < pr.world; q++)
      acc += *reinterpret_cast<volatile int*>(&pr.slots[pr.rank][(q * 2 + par) * 32 + lane]);
    out = __int_as_float(ok ? acc : -1);
  }
  __syncwarp();
  if (lane == 0) *pr.seq_counter = seq;
  return out;
}

// stand-alone form: all-reduce n <= 32 ints in place (per-sweep counts of the sharded map)
__global__ void peer_allreduce_ints_kernel(PeerReduce pr, int* data, int n) {
  if (blockIdx.x != 0 || threadIdx.x >= 32) return;
  const int lane = threadIdx.x;
  const float v = __int_as_float(lane < n ? data[lane] : 0);
  const float r = peer_allreduce32<1>(pr, v);
  if (lane < n) data[lane] = __float_as_int(r);
}

// block reduction of NEQ accumulators -> partials[block]; the last block to finish folds all partials in block
// order (double accumulation) into result[NEQ] and resets the ticket for the next launch.
__device__ __forceinline__ bool reduce_normal_equations(float* acc, float* __restrict__ partials,
                                                        float* __restrict__ result, unsigned int* ticket,
                                                        ResultMailbox mb, unsigned n_blocks) {
  __shared__ float s_part[LM_THREADS / 32][NEQ];
  __shared__ bool s_last;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < 29; k++) {
    float v = acc[k];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (lane == 0) s_part[warp][k] = v;
  }
  __syncthreads();
  if (threadIdx.x < NEQ) {
    float v = 0.f;
    if (threadIdx.x < 29)
      for (int wv = 0; wv < LM_THREADS / 32; wv++) v += s_part[wv][threadIdx.x];
    __stcg(&partials[(size_t)blockIdx.x * NEQ + threadIdx.x], v);
  }
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) s_last = (atomicAdd(ticket, 1u) == n_blocks - 1);
  __syncthreads();
  if (s_last) {
    __threadfence();
    // fixed summation order -> run-to-run deterministic: warp w folds blocks w, w+4, w+8, ... in double, then the four
    // warp sums are added in warp order
    __shared__ double s_fold[LM_THREADS / 32][NEQ];
    {
      double v = 0.0;
      for (unsigned bk = warp; bk < n_blocks; bk += LM_THREADS / 32) v += (double)__ldcg(&partials[(size_t)bk * NEQ + lane]);
      s_fold[warp][lane] = v;
    }
    __syncthreads();
    if (threadIdx.x < NEQ) {
      double v = 0.0;
      for (int wv = 0; wv < LM_THREADS / 32; wv++) v += s_fold[wv][threadIdx.x];
      result[threadIdx.x] = (float)v;
      mailbox_post_value(mb, threadIdx.x, (float)v);
    }
    if (threadIdx.x == 0) *ticket = 0u;
    __syncthreads();
    mailbox_post_seq(mb);
  }
  return s_last;
}

constexpr int MAP_THREADS = 256;
constexpr int MAP_GROUP = 8;                          // lanes per query in the search phase
constexpr int MAP_Q_PER_BLOCK = MAP_THREADS / MAP_GROUP;
static_assert(MAP_Q_PER_BLOCK == 32, "the fit phase maps one query to one lane of warp 0");

// Two phases per CTA of 32 queries (with the fit done by lane 0 of every 8-lane group, a third of all warp instructions
// ran at 4 / 32 lanes):
//   search : 8 warps, 8 lanes per query -> five neighbours per query in shared memory
//   fit    : warp 0, one query per lane -> line / plane fit, Jacobian row, warp-shuffle reduction of the 29 sums,
//            partial written straight from registers; the last CTA folds all partials in fixed order.
// 64 registers / thread -> 4 CTAs per SM: 528 CTAs resident at once on the 132 SMs of an H100, about the ~550 CTAs
// of an HDL-64 sweep (with fewer CTAs per SM a second, mostly empty wave costs as much as the first).
// MLP = candidate loads in flight per lane.  On the HBM-bound 20 M-point stress, MLP 4 (80 registers, 3 CTAs / SM) and
// MLP 8 (96 registers, 2 CTAs) were slower than MLP 2 (64 registers, 4 CTAs / SM): occupancy is worth more than deeper
// per-lane pipelining, so 2 is used everywhere.
template <bool STATS, typename LOOKUP, bool DEVLOOP = false, int MLP = 2>
__global__ void __launch_bounds__(MAP_THREADS, MLP > 4 ? 2 : (MLP > 2 ? 3 : 4))
map_iterate_kernel(LOOKUP corner_grid, LOOKUP surf_grid, const float4* queries, const float4* queries_surf,
                   int n_corner_total, int c0, int n_corner, int s0, int n_surf, int corner_blocks, MapIterArgs a_param,
                   float* __restrict__ partials, float* __restrict__ result, unsigned int* ticket,
                   float4* __restrict__ dbg_coeff, int8_t* __restrict__ dbg_sel,
                   unsigned long long* __restrict__ walk_totals, const MapLmState* __restrict__ lm = nullptr,
                   ResultMailbox mb = ResultMailbox{nullptr, 0}, ShardSpec sh = ShardSpec{0, 1, 0},
                   PeerReduce pr = PeerReduce{}) {
  // DEVLOOP (device-resident loop, lmstep.cuh): the arguments of the current iteration come from the state block
  // (staged in shared memory; the by-value `a_param` of the per-iteration API stays in the constant bank), and there
  // is nothing to do once the loop has converged
  __shared__ MapIterArgs s_args;
  __shared__ alignas(16) unsigned char s_lookup[DEVLOOP ? MAP_LOOKUP_BYTES : 16];
  unsigned n_blocks = gridDim.x;
  if (DEVLOOP) {
    if (lm->h.done) return;
    const MapLoopIo& io = lm->io;  // uniform loads; the grid of the loop graph is sized for a capacity
    n_blocks = (unsigned)io.n_blocks;
    if (blockIdx.x >= n_blocks) return;
    if (threadIdx.x < (int)(sizeof(MapIterArgs) / 4))
      reinterpret_cast<float*>(&s_args)[threadIdx.x] = reinterpret_cast<const float*>(&lm->args)[threadIdx.x];
    queries = io.queries; queries_surf = io.queries_surf; n_corner_total = io.n_corner_total; c0 = io.c0;
    n_corner = io.n_corner; s0 = io.s0; n_surf = io.n_surf; corner_blocks = io.corner_blocks;
    static_assert(sizeof(LOOKUP) <= MAP_LOOKUP_BYTES, "lookup does not fit its slot in MapLoopIo");
    const int kind = (int)blockIdx.x < corner_blocks ? 0 : 1;
    if (threadIdx.x < (int)((sizeof(LOOKUP) + 3) / 4))
      reinterpret_cast<unsigned*>(s_lookup)[threadIdx.x] = reinterpret_cast<const unsigned*>(io.lookup[kind])[threadIdx.x];
    __syncthreads();
  }
  const MapIterArgs& a = DEVLOOP ? s_args : a_param;
  __shared__ float4 s_nn[MAP_Q_PER_BLOCK][5];                 // xyz of the five neighbours, w = index bits (< 0: none)
  __shared__ unsigned s_pre[MAP_Q_PER_BLOCK][GRID_SLOTS + 1];
  __shared__ unsigned s_first[MAP_Q_PER_BLOCK][GRID_SLOTS];
  __shared__ bool s_last;

  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, sub = lane & (MAP_GROUP - 1);
  const unsigned gmask = 0xffu << (lane & ~(MAP_GROUP - 1));
  const bool is_corner = (int)blockIdx.x < corner_blocks;
  const int block_first = (is_corner ? blockIdx.x : blockIdx.x - corner_blocks) * MAP_Q_PER_BLOCK;
  const int n_kind = is_corner ? n_corner : n_surf;
  // this rank's slice: corners [c0, c0 + n_corner), surfaces [s0, s0 + n_surf) (the whole range on one GPU)
  const int q_base = is_corner ? c0 : n_corner_total + s0;   // index in the concatenated numbering (debug outputs)
  const float4* __restrict__ qsrc = is_corner ? queries + c0 : queries_surf + s0;
  // cell -> run of map points (gridnn.cuh / mapstore.cuh)
  LOOKUP grid = DEVLOOP ? *reinterpret_cast<const LOOKUP*>(s_lookup) : (is_corner ? corner_grid : surf_grid);

  {  // ---- search: 8 lanes per query
    const int g = threadIdx.x / MAP_GROUP;
    const int local = block_first + g;
    if (local < n_kind) {  // uniform within a group of 8 lanes
      const float4 po = qsrc[local];
      float sx, sy, sz;
      associate_to_map(a, po, sx, sy, sz);
      Cand5 best;
#pragma unroll
      for (int i = 0; i < 5; i++) { best.d[i] = 1.0f; best.id[i] = -1; }
      // cube-sharded map: the rank owning the cell of the transformed point evaluates it, everybody else skips it
      if (shard_owns(sh, store_cell(sx))) {
        unsigned ws[2] = {0u, 0u};
        grid_knn5_group8<STATS, LOOKUP, MLP>(grid, sx, sy, sz, sub, gmask, s_pre[g], s_first[g], best, ws);
        if (STATS) {
          atomicAdd(&walk_totals[0], (unsigned long long)ws[0]);
          atomicAdd(&walk_totals[1], (unsigned long long)ws[1]);
        }
      }
      if (sub < 5) {  // lanes 0..4 fetch one neighbour each
        const int id = sub == 0 ? best.id[0] : sub == 1 ? best.id[1] : sub == 2 ? best.id[2] : sub == 3 ? best.id[3]
                                                                                                       : best.id[4];
        float4 p = make_float4(0.f, 0.f, 0.f, 0.f);
        if (id >= 0) p = __ldg(&grid.points()[id]);
        p.w = __int_as_float(id);
        s_nn[g][sub] = p;
      }
    }
  }
  __syncthreads();

  if (warp == 0) {  // ---- fit: one query per lane
    const int local = block_first + lane;
    float row[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f}, rhs = 0.f;
    bool sel = false;
    if (local < n_kind) {
      const int qi = q_base + local;
      const float4 po = qsrc[local];
      float sx, sy, sz;
      associate_to_map(a, po, sx, sy, sz);
      Top5 nn;
#pragma unroll
      for (int j = 0; j < 5; j++) {
        const float4 p = s_nn[lane][j];
        nn.x[j] = p.x; nn.y[j] = p.y; nn.z[j] = p.z;
        nn.idx[j] = __float_as_int(p.w);
        nn.d[j] = 0.f;
      }
      float4 coeff = make_float4(0.f, 0.f, 0.f, 0.f);
      sel = is_corner ? corner_fit(nn, sx, sy, sz, coeff) : surf_fit(nn, sx, sy, sz, coeff);
      if (dbg_coeff) {
        dbg_coeff[qi] = coeff;
        dbg_sel[qi] = sel ? 1 : 0;
      }
      if (sel) map_jacobian_row(a, po, coeff, row, rhs);
    }
    // 21 + 6 + 2 sums over the warp; after the xor butterfly every lane holds every sum, lane k keeps sum k
    float mine = 0.f;
    int k = 0;
#pragma unroll
    for (int i = 0; i < 6; i++)
#pragma unroll
      for (int j = i; j < 6; j++) {
        float v = row[i] * row[j];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if (lane == k) mine = v;
        k++;
      }
#pragma unroll
    for (int i = 0; i < 6; i++) {
      float v = row[i] * rhs;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
      if (lane == 21 + i) mine = v;
    }
    {
      const unsigned sel_mask = __ballot_sync(0xffffffffu, sel);
      if (lane == 27) mine = (float)__popc(sel_mask);
      if (lane == 28) mine = is_corner ? (float)__popc(sel_mask) : 0.f;
    }
    __stcg(&partials[(size_t)blockIdx.x * NEQ + lane], mine);
    __threadfence();
    __syncwarp();
    if (lane == 0) s_last = (atomicAdd(ticket, 1u) == n_blocks - 1);
  }
  __syncthreads();
  if (s_last) {
    // the last CTA folds all partials: warp w takes CTAs w, w+8, ... (eight independent loads in flight) in double,
    // then the eight warp sums are added in warp order -> run-to-run deterministic
    __threadfence();
    __shared__ double s_fold[MAP_THREADS / 32][NEQ];
    constexpr unsigned NW = MAP_THREADS / 32;
    const unsigned nb = n_blocks;
    double v = 0.0;
    unsigned bk = warp;
    for (; bk + 7 * NW < nb; bk += 8 * NW) {
      float t[8];
#pragma unroll
      for (int u = 0; u < 8; u++) t[u] = __ldcg(&partials[(size_t)(bk + u * NW) * NEQ + lane]);
#pragma unroll
      for (int u = 0; u < 8; u++) v += (double)t[u];
    }
    for (; bk < nb; bk += NW) v += (double)__ldcg(&partials[(size_t)bk * NEQ + lane]);
    s_fold[warp][lane] = v;
    __syncthreads();
    if (threadIdx.x < NEQ) {
      double r = 0.0;
      for (unsigned wv = 0; wv < NW; wv++) r += s_fold[wv][threadIdx.x];
      float rf = (float)r;
      if (pr.world > 1) rf = peer_allreduce32<0>(pr, rf);  // fused all-reduce over NVLink peer memory (warp 0)
      result[threadIdx.x] = rf;
      mailbox_post_value(mb, threadIdx.x, rf);
    }
    if (threadIdx.x == 0) *ticket = 0u;
    __syncthreads();
    mailbox_post_seq(mb);
  }
}

__global__ void map_lm_step_kernel(MapLmState* st, const float* __restrict__ result, unsigned long long handle = 0ull,
                                   float* mailbox_host = nullptr) {
  __shared__ float s_r[NEQ];  // see odom_lm_step_kernel
  if (blockIdx.x != 0 || threadIdx.x >= 32) return;
  s_r[threadIdx.x] = __ldcg(&result[threadIdx.x]);
  __syncwarp();
  if (!st->h.done) map_lm_step_warp(st, s_r);  // uniform over the warp
  if (threadIdx.x == 0) lm_loop_control(st->h, handle, mailbox_host);
}

}  // namespace loamb
