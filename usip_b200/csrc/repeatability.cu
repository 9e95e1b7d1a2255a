// repeatability.cu -- keypoint repeatability of evaluation/matlab/eval_repeatability/eval_rep.m:142-146 for a whole
// keypoint-count sweep in one launch.
//
// eval_rep.m reads each pair's two keypoint files, maps both to the ground-truth frame and counts the anchor keypoints
// whose nearest positive keypoint lies within the inlier radius.  Every K of a sweep reads a prefix of the same
// selection order, so one pass over the positive prefix serves all of them: every anchor keypoint keeps a running
// minimum over the positives and reads it off at each K boundary.
//
// Arithmetic: fp64 with a fixed order and no contraction, so that a float64 restatement on the host (tests/rep_ref.py)
// reproduces every count exactly.  Minimum over squared distances, then one sqrt: a correctly rounded sqrt is monotone,
// so this is the minimum of the distances bit for bit.
#include "common.cuh"

namespace usip {

constexpr int REP_THREADS = 256;

struct RepKs { int32_t k[USIP_REP_MAX_K]; };

// ((m0*x + m1*y) + m2*z) + m3 for the three rows of a row-major 3x4 map
__device__ __forceinline__ void rep_map(const double* T, double& x, double& y, double& z) {
  const double a = x, b = y, c = z;
  x = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(T[0], a), __dmul_rn(T[1], b)), __dmul_rn(T[2], c)), T[3]);
  y = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(T[4], a), __dmul_rn(T[5], b)), __dmul_rn(T[6], c)), T[7]);
  z = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(T[8], a), __dmul_rn(T[9], b)), __dmul_rn(T[10], c)), T[11]);
}

// one CTA per pair; shared memory: L anchor and L positive keypoints, SoA fp64 (L = min(M, largest K))
__global__ void __launch_bounds__(REP_THREADS)
repeatability_kernel(const float* __restrict__ kp, const int32_t* __restrict__ order,
                     const int32_t* __restrict__ count, int M, int L, const int32_t* __restrict__ pairs,
                     const double* __restrict__ frames, RepKs ks, int nK, double radius, int32_t* __restrict__ inliers,
                     int32_t* __restrict__ n_anc) {
  extern __shared__ __align__(16) double rep_smem[];
  __shared__ int32_t s_cnt[USIP_REP_MAX_K];
  double* ax = rep_smem;
  double* ay = ax + L;
  double* az = ay + L;
  double* px = az + L;
  double* py = px + L;
  double* pz = py + L;
  const int p = blockIdx.x, tid = threadIdx.x;
  const int sa = pairs[2 * p], sp = pairs[2 * p + 1];
  const int na = min(count[sa], L), np = min(count[sp], L);
  const double* F = frames + (int64_t)p * 36;     // F_a, F_p, T_gt

  if (tid < nK) s_cnt[tid] = 0;
  for (int i = tid; i < na; i += blockDim.x) {
    const int j = order[(int64_t)sa * M + i];
    const float* q = kp + (int64_t)sa * 3 * M + j;
    double x = q[0], y = q[M], z = q[2 * M];
    rep_map(F, x, y, z);
    ax[i] = x; ay[i] = y; az[i] = z;
  }
  for (int i = tid; i < np; i += blockDim.x) {
    const int j = order[(int64_t)sp * M + i];
    const float* q = kp + (int64_t)sp * 3 * M + j;
    double x = q[0], y = q[M], z = q[2 * M];
    rep_map(F + 12, x, y, z);
    rep_map(F + 24, x, y, z);
    px[i] = x; py[i] = y; pz[i] = z;
  }
  __syncthreads();

  // na is the same for the whole CTA, so every thread runs the same iterations and the ballots see full warps
  const int lane = tid & 31;
  for (int i0 = 0; i0 < na; i0 += blockDim.x) {
    const int i = i0 + tid;
    const bool live = i < na;
    const double x = live ? ax[i] : 0.0, y = live ? ay[i] : 0.0, z = live ? az[i] : 0.0;
    double m = __longlong_as_double(0x7ff0000000000000ll);     // +inf
    int j = 0;
    for (int k = 0; k < nK; ++k) {
      const int npk = min(ks.k[k], np);
      for (; j < npk; ++j) {
        const double dx = __dadd_rn(px[j], -x), dy = __dadd_rn(py[j], -y), dz = __dadd_rn(pz[j], -z);
        const double s = __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
        m = fmin(m, s);
      }
      const bool in = live && i < ks.k[k] && __dsqrt_rn(m) < radius;
      const unsigned b = __ballot_sync(0xffffffffu, in);
      if (lane == 0 && b) atomicAdd(&s_cnt[k], __popc(b));
    }
  }
  __syncthreads();
  if (tid < nK) {
    inliers[(int64_t)p * nK + tid] = s_cnt[tid];
    n_anc[(int64_t)p * nK + tid] = min(ks.k[tid], na);
  }
}

}  // namespace usip

using namespace usip;

extern "C" int usip_repeatability_f64(const float* keypoints, const int32_t* order, const int32_t* count, int n_scans,
                                      int M, const int32_t* pairs, const double* frames, int P, const int32_t* ks,
                                      int nK, double radius, int32_t* inliers, int32_t* n_anc, void* stream) {
  USIP_REQUIRE(keypoints && order && count && pairs && frames && ks && inliers && n_anc, "repeatability: null pointer");
  USIP_REQUIRE(n_scans > 0 && M > 0 && P > 0, "repeatability: bad sizes");
  USIP_REQUIRE(nK >= 1 && nK <= USIP_REP_MAX_K, "repeatability: 1 to USIP_REP_MAX_K keypoint counts");
  RepKs k;
  for (int i = 0; i < nK; ++i) {
    USIP_REQUIRE(ks[i] > 0 && (i == 0 || ks[i] > ks[i - 1]), "repeatability: keypoint counts must ascend and be > 0");
    k.k[i] = ks[i];
  }
  USIP_REQUIRE(radius > 0.0, "repeatability: the inlier radius must be > 0");
  const int L = min(M, ks[nK - 1]);
  USIP_REQUIRE(L <= USIP_REP_MAX_KEYPOINTS, "repeatability: more keypoints per scan than shared memory holds");
  const int smem = 6 * L * (int)sizeof(double);
  cudaError_t e = cudaFuncSetAttribute(repeatability_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  if (e != cudaSuccess) { set_last_error("repeatability: smem attribute"); return (int)e; }
  repeatability_kernel<<<P, REP_THREADS, smem, (cudaStream_t)stream>>>(keypoints, order, count, M, L, pairs, frames, k,
                                                                        nK, radius, inliers, n_anc);
  return check_launch("repeatability_kernel");
}
