// nms.cu -- inference post-processing (SURVEY section 8 f-3): sigma-ordered radius non-maximum suppression of the
// detector's keypoints.
//
// Reference: evaluation/save_keypoints.py:180-216 nms(): repeat { take the remaining keypoint with the smallest sigma
// (np.argmin: first minimum), emit it, drop every remaining keypoint whose float32 np.linalg.norm distance to it is not
// > NMS_radius }.  Equivalent single sweep: visit the keypoints in (sigma, index) order, NaN sigmas first, and emit the
// ones no earlier emitted keypoint has suppressed.  One CTA per cloud; the sweep is sequential in the keypoints, parallel in the
// suppression test.  Distances use the repository's fp32 policy (sqdist_rn + correctly rounded sqrt == numpy).
#include "common.cuh"

namespace usip {

constexpr int NMS_THREADS = 1024;

__global__ void __launch_bounds__(NMS_THREADS)
nms_kernel(const float* __restrict__ kp, const float* __restrict__ sigma, float radius, int32_t* __restrict__ out_idx,
           int32_t* __restrict__ out_count, int M) {
  extern __shared__ float nms_sm[];                 // x[M] y[M] z[M] sigma[M] | order[M] (int) | alive[M] (int)
  float* sx = nms_sm; float* sy = sx + M; float* sz = sy + M; float* ss = sz + M;
  int* order = reinterpret_cast<int*>(ss + M);
  int* alive = order + M;
  __shared__ int s_count;
  const int b = blockIdx.x, tid = threadIdx.x;
  const float* p = kp + (size_t)b * 3 * M;          // (B, 3, M): the detector's output layout
  int32_t* o = out_idx + (size_t)b * M;
  for (int i = tid; i < M; i += NMS_THREADS) {
    sx[i] = p[i]; sy[i] = p[M + i]; sz[i] = p[2 * M + i]; ss[i] = sigma[(size_t)b * M + i];
    alive[i] = 1; o[i] = -1;
  }
  if (tid == 0) s_count = 0;
  __syncthreads();
  if (radius < 0.01f) {                             // save_keypoints.py:187-188: pass-through, input order
    for (int i = tid; i < M; i += NMS_THREADS) o[i] = i;
    if (tid == 0) out_count[b] = M;
    return;
  }
  // rank by (sigma, index): the order in which repeated first-arg-min would visit the keypoints.  np.argmin returns the
  // first NaN when there is one, so NaN sigmas come before every finite one, in index order among themselves; the ranks
  // are then a permutation of 0..M-1 and every order[] slot is written.
  for (int i = tid; i < M; i += NMS_THREADS) {
    const float si = ss[i];
    const bool ni = si != si;
    int rk = 0;
    for (int j = 0; j < M; ++j) {
      const float sj = ss[j];
      const bool nj = sj != sj;
      rk += (ni ? (nj && j < i) : (nj || sj < si || (sj == si && j < i))) ? 1 : 0;
    }
    order[rk] = i;
  }
  __syncthreads();
  for (int s = 0; s < M; ++s) {
    const int i = order[s];
    if (!alive[i]) continue;                        // uniform: alive[] only changes between barriers
    const float cx = sx[i], cy = sy[i], cz = sz[i];
    __syncthreads();                                // everyone has read alive[i] before it is cleared below
    if (tid == 0) { o[s_count] = i; s_count += 1; }
    for (int j = tid; j < M; j += NMS_THREADS)
      if (alive[j] && !(__fsqrt_rn(sqdist_rn(cx, cy, cz, sx[j], sy[j], sz[j])) > radius)) alive[j] = 0;
    __syncthreads();
  }
  if (tid == 0) out_count[b] = s_count;
}

}  // namespace usip

using namespace usip;

extern "C" int usip_nms_f32(const float* keypoints, const float* sigmas, float radius, int32_t* out_idx,
                            int32_t* out_count, int B, int M, void* stream) {
  USIP_REQUIRE(keypoints && sigmas && out_idx && out_count && B > 0 && M > 0, "nms: bad args");
  const size_t smem = (size_t)M * 6 * sizeof(float);
  USIP_REQUIRE(smem <= 200 * 1024, "nms: M too large");
  if (smem > 40 * 1024) cudaFuncSetAttribute(nms_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  nms_kernel<<<B, NMS_THREADS, smem, (cudaStream_t)stream>>>(keypoints, sigmas, radius, out_idx, out_count, M);
  return check_launch("nms_kernel");
}
