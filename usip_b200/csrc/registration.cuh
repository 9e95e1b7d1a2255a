// registration.cuh -- the fp64 helpers that registration.cu (RANSAC) and fgr.cu (Fast Global Registration) share: the
// inlier test, the information matrix's A columns and an order-keeping block rank.  No contraction anywhere.
#pragma once
#include "common.cuh"

namespace usip {

struct RegKs { int32_t k[USIP_REP_MAX_K]; };
// the keypoint-count sweep of the registration entry points: 1..USIP_REP_MAX_K ascending positive values (host)
int reg_check_ks(const int32_t* ks, int nK, RegKs& k);

__device__ __forceinline__ double dsub(double a, double b) { return __dadd_rn(a, -b); }

// ||x1 - (R x2 + t)|| < thr, each row ((R0 x + R1 y) + R2 z) + t, then ((dx^2 + dy^2) + dz^2), sqrt
__device__ __forceinline__ bool reg_inlier(const double* Rt, double ax, double ay, double az, double px, double py,
                                           double pz, double thr) {
  const double ex = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(Rt[0], px), __dmul_rn(Rt[1], py)), __dmul_rn(Rt[2], pz)), Rt[3]);
  const double ey = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(Rt[4], px), __dmul_rn(Rt[5], py)), __dmul_rn(Rt[6], pz)), Rt[7]);
  const double ez = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(Rt[8], px), __dmul_rn(Rt[9], py)), __dmul_rn(Rt[10], pz)), Rt[11]);
  const double dx = dsub(ax, ex), dy = dsub(ay, ey), dz = dsub(az, ez);
  return __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz))) < thr;
}

// Column k of register2Fragments.m's A = [I3 | [[0, 2z, -2y], [-2z, 0, 2x], [2y, -2x, 0]]] at (x, y, z)
__device__ __forceinline__ void reg_info_col(int k, double x, double y, double z, double a[3]) {
  const double x2 = __dmul_rn(2.0, x), y2 = __dmul_rn(2.0, y), z2 = __dmul_rn(2.0, z);
  a[0] = k == 0 ? 1.0 : k == 4 ? z2 : k == 5 ? -y2 : 0.0;
  a[1] = k == 1 ? 1.0 : k == 3 ? -z2 : k == 5 ? x2 : 0.0;
  a[2] = k == 2 ? 1.0 : k == 3 ? y2 : k == 4 ? -x2 : 0.0;
}

// Entry (r, c) of A^T A at (x, y, z): ((A0r A0c + A1r A1c) + A2r A2c)
__device__ __forceinline__ double reg_info_entry(int r, int c, double x, double y, double z) {
  double ar[3], ac[3];
  reg_info_col(r, x, y, z, ar);
  reg_info_col(c, x, y, z, ac);
  return __dadd_rn(__dadd_rn(__dmul_rn(ar[0], ac[0]), __dmul_rn(ar[1], ac[1])), __dmul_rn(ar[2], ac[2]));
}

// Exclusive rank of this thread's flag among the block's set flags, in thread order; *total gets the block's count.
// warp_tot holds blockDim / 32 ints of shared memory.  Every thread of the block must call it (two barriers).
__device__ __forceinline__ int reg_block_rank(bool f, int* warp_tot, int* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  const uint32_t b = __ballot_sync(0xffffffffu, f);
  if (lane == 0) warp_tot[warp] = __popc(b);
  __syncthreads();
  int before = 0, all = 0;
  for (int w = 0; w < nw; ++w) {
    const int c = warp_tot[w];
    before += w < warp ? c : 0;
    all += c;
  }
  __syncthreads();
  *total = all;
  return before + __popc(b & ((1u << lane) - 1u));
}

}  // namespace usip
