// fps.cu -- farthest point sampling of the SOM nodes (SURVEY section 8 f-2): the step immediately before the hot path.
//
// Reference: data/kitti_detector_loader.py:68-83 (FarthestSampler), called per cloud in the DataLoader workers on a
// random N/3 subset (:144-145).  numpy semantics reproduced bit for bit: the running "distance to the chosen set" is
// float64 ((p0 - p)**2).sum(axis=1) with p0 a float64 copy of a float32 point, i.e. ((dx*dx + dy*dy) + dz*dz) in double
// without FMA; np.argmax returns the FIRST maximum; np.minimum keeps the smaller value.
//
// One CTA per cloud: every thread owns its points (strided, so indices ascend inside a thread) and keeps their running
// minima in registers; an iteration is a distance update + a block-wide (value, first index) arg-max: warp shuffles,
// one round through shared memory, two barriers.
//
// usip_fps_f64 is the same kernel on float64 points: data/scenenn_descriptor_loader.py's FarthestSampler runs on the
// float64 ICP'd anchor.  Only where a thread's points live differs: float32 points sit in registers; 8 x 3 doubles
// would take 48 of the 64 registers a 1024-thread CTA may use, so float64 points sit in shared memory (three planes of
// Ns doubles, at most 192 KB) and are read where they are used.
#include "common.cuh"

namespace usip {

constexpr int FPS_THREADS = 1024;
constexpr int FPS_PPT = 8;                        // points per thread -> Ns <= 8192 per cloud

template <typename T>
__device__ __forceinline__ double fps_d2(double sx, double sy, double sz, T x, T y, T z) {
  const double dx = __dsub_rn(sx, (double)x), dy = __dsub_rn(sy, (double)y), dz = __dsub_rn(sz, (double)z);
  return __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
}

template <typename T>
__global__ void __launch_bounds__(FPS_THREADS)
fps_kernel(const T* __restrict__ pts, const int32_t* __restrict__ start, int32_t* __restrict__ out_idx,
           float* __restrict__ out_nodes, int Ns, int k) {
  __shared__ double wval[32];
  __shared__ int widx[32];
  __shared__ int s_sel;
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  const T* p = pts + (size_t)b * Ns * 3;          // (Ns, 3) row-major, like the numpy array the reference samples from
  constexpr bool in_regs = sizeof(T) == sizeof(float);
  extern __shared__ double fps_smem[];            // float64 points: x, y and z planes of Ns doubles
  float px[FPS_PPT], py[FPS_PPT], pz[FPS_PPT];    // float32 points
  if constexpr (in_regs) {
#pragma unroll
    for (int j = 0; j < FPS_PPT; ++j) {
      const int i = tid + j * FPS_THREADS;
      px[j] = py[j] = pz[j] = 0.f;
      if (i < Ns) { px[j] = p[3 * i]; py[j] = p[3 * i + 1]; pz[j] = p[3 * i + 2]; }
    }
  } else {
    for (int i = tid; i < Ns; i += FPS_THREADS) {
      fps_smem[i] = p[3 * i]; fps_smem[Ns + i] = p[3 * i + 1]; fps_smem[2 * Ns + i] = p[3 * i + 2];
    }
    __syncthreads();
  }
  double md[FPS_PPT];
  int sel = start[b];
  for (int it = 0; it < k; ++it) {
    const double sx = (double)p[3 * sel], sy = (double)p[3 * sel + 1], sz = (double)p[3 * sel + 2];
    if (tid == 0) {
      out_idx[(size_t)b * k + it] = sel;
      if (out_nodes) {                              // (B, 3, k): the detector's node layout
        out_nodes[((size_t)b * 3 + 0) * k + it] = (float)sx;
        out_nodes[((size_t)b * 3 + 1) * k + it] = (float)sy;
        out_nodes[((size_t)b * 3 + 2) * k + it] = (float)sz;
      }
    }
    if (it == k - 1) break;
    // distance update + thread-local first arg-max
    double bv = -1.0; int bi = 0x7fffffff;
#pragma unroll
    for (int j = 0; j < FPS_PPT; ++j) {
      const int i = tid + j * FPS_THREADS;
      if (i < Ns) {
        const double d = in_regs ? fps_d2(sx, sy, sz, px[j], py[j], pz[j])
                                 : fps_d2(sx, sy, sz, fps_smem[i], fps_smem[Ns + i], fps_smem[2 * Ns + i]);
        md[j] = (it == 0) ? d : (d < md[j] ? d : md[j]);
        if (md[j] > bv) { bv = md[j]; bi = i; }     // indices ascend with j: '>' keeps the first maximum
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const double ov = __shfl_xor_sync(0xffffffffu, bv, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
    }
    if (lane == 0) { wval[w] = bv; widx[w] = bi; }
    __syncthreads();
    if (w == 0) {
      bv = wval[lane]; bi = widx[lane];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const double ov = __shfl_xor_sync(0xffffffffu, bv, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
      }
      if (lane == 0) s_sel = bi;
    }
    __syncthreads();
    sel = s_sel;
  }
}

}  // namespace usip

using namespace usip;

extern "C" int usip_fps_f32(const float* pts, const int32_t* start, int32_t* out_idx, float* out_nodes, int B, int Ns,
                            int k, void* stream) {
  USIP_REQUIRE(pts && start && out_idx && B > 0 && Ns > 0 && k > 0, "fps: bad args");
  USIP_REQUIRE(Ns <= FPS_THREADS * FPS_PPT, "fps: at most 8192 candidate points per cloud");
  fps_kernel<float><<<B, FPS_THREADS, 0, (cudaStream_t)stream>>>(pts, start, out_idx, out_nodes, Ns, k);
  return check_launch("fps_kernel");
}

extern "C" int usip_fps_f64(const double* pts, const int32_t* start, int32_t* out_idx, float* out_nodes, int B, int Ns,
                            int k, void* stream) {
  USIP_REQUIRE(pts && start && out_idx && B > 0 && Ns > 0 && k > 0, "fps_f64: bad args");
  USIP_REQUIRE(Ns <= FPS_THREADS * FPS_PPT, "fps_f64: at most 8192 candidate points per cloud");
  const int smem = 3 * Ns * (int)sizeof(double);
  cudaError_t e = cudaFuncSetAttribute(fps_kernel<double>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  if (e != cudaSuccess) { set_last_error("fps_f64: smem attribute"); return (int)e; }
  fps_kernel<double><<<B, FPS_THREADS, smem, (cudaStream_t)stream>>>(pts, start, out_idx, out_nodes, Ns, k);
  return check_launch("fps_kernel<double>");
}
