// common.cuh -- shared helpers for libusip_b200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <math.h>
#include "../../include/usip_b200.h"

namespace usip {

void set_last_error(const char* what);

inline int check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) { set_last_error(what); return (int)e; }
  return 0;
}
inline int fail(const char* what) { set_last_error(what); return -1; }

#define USIP_REQUIRE(cond, msg) do { if (!(cond)) return ::usip::fail(msg); } while (0)

// multiprocessor count of the current device (queried once: launch sizes are per SM)
inline int device_sm_count() {
  static int sm_count = 0;
  if (sm_count == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sm_count, cudaDevAttrMultiProcessorCount, dev);
  }
  return sm_count;
}

__host__ __device__ inline int cdiv(int a, int b) { return (a + b - 1) / b; }
__host__ __device__ inline int64_t cdiv64(int64_t a, int64_t b) { return (a + b - 1) / b; }

// Order-preserving float -> uint32 map (total order, -0 < +0; NaN handled by callers).
__device__ __forceinline__ uint32_t f2ord(float f) {
  uint32_t u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float ord2f(uint32_t o) {
  uint32_t u = (o & 0x80000000u) ? (o & 0x7fffffffu) : ~o;
  return __uint_as_float(u);
}

// Squared distance with the reference's exact fp32 op order (no FMA contraction):
// (dx*dx + dy*dy) + dz*dz   -- util/som.py:35-36, torch.norm at networks.py:357, losses.py:66.
__device__ __forceinline__ float sqdist_rn(float ax, float ay, float az, float bx, float by, float bz) {
  float dx = __fsub_rn(ax, bx), dy = __fsub_rn(ay, by), dz = __fsub_rn(az, bz);
  return __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
}

// ((m0*x + m1*y) + m2*z) + m3 for the three rows of a row-major 3x4 map, fp64 without contraction (repeatability.cu's
// order); registration.cu and overlap.cu map points with it.
__device__ __forceinline__ void reg_map(const double* T, double& x, double& y, double& z) {
  const double a = x, b = y, c = z;
  x = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(T[0], a), __dmul_rn(T[1], b)), __dmul_rn(T[2], c)), T[3]);
  y = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(T[4], a), __dmul_rn(T[5], b)), __dmul_rn(T[6], c)), T[7]);
  z = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(T[8], a), __dmul_rn(T[9], b)), __dmul_rn(T[10], c)), T[11]);
}

// Philox4x32-10 (Salmon et al., SC'11): counter c, key (k0, k1) -> four random words.  pairgen.cu and registration.cu
// build their counters from it.
__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint32_t k0, uint32_t k1) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t hi0 = __umulhi(0xD2511F53u, c.x), lo0 = 0xD2511F53u * c.x;
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, c.z), lo1 = 0xCD9E8D57u * c.z;
    c = make_uint4(hi1 ^ c.y ^ k0, lo1, hi0 ^ c.w ^ k1, lo0);
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  return c;
}

// Counter layout of every per-point stream of pairgen.cu and handcrafted.cu: (item, cloud, step, purpose | sub << 8 |
// step_hi << 16), key (seed_lo, seed_hi).  One purpose value per stream, so that no two streams share a counter.
enum { PURPOSE_ROWS = 0, PURPOSE_CAND = 1, PURPOSE_START = 2, PURPOSE_JIT_PC = 3, PURPOSE_JIT_SN = 4,
       PURPOSE_JIT_NODE = 5, PURPOSE_NOISE = 6, PURPOSE_HC_KEYPOINT = 7, PURPOSE_HC_PAD = 8 };

__device__ __forceinline__ uint4 pg_random(uint64_t seed, uint64_t step, int cloud, int item, int purpose, int sub) {
  const uint4 ctr = make_uint4((uint32_t)item, (uint32_t)cloud, (uint32_t)step,
                               (uint32_t)purpose | ((uint32_t)sub << 8) | ((uint32_t)(step >> 32) << 16));
  return philox4x32_10(ctr, (uint32_t)seed, (uint32_t)(seed >> 32));
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

}  // namespace usip
