// optim.cu -- the parameter update of the train step: Adam over ONE flat fp32 buffer.
//
// Replaces torch.optim.Adam(detector.parameters(), lr, betas=(0.9, 0.999), weight_decay=0) of the reference
// (models/keypoint_detector.py:42-45, keypoint_descriptor.py:32-35) -- a dozen foreach launches over 42 tensors -- by
// one launch over the flat parameter / gradient / moment buffers the host side keeps (usip_b200/optim.py).  The step
// counter and the learning rate live in DEVICE memory so that the launch can sit inside a CUDA graph: the kernel reads
// step t-1, updates with the bias corrections of step t, and the last CTA to arrive publishes t.
// The update is torch's Adam in fp32, m = b1 m + (1-b1) g;  v = b2 v + (1-b2) g^2;
// p -= (lr / (1-b1^t)) * m / (sqrt(v) / sqrt(1-b2^t) + eps), but not its exact rounding: torch's single-tensor path
// updates m as a lerp, m + (1-b1)(g - m), and divides by sqrt(1-b2^t), where this kernel forms b1 m + (1-b1) g and
// multiplies by a (double-rounded) 1/sqrt(1-b2^t).  The betas arrive as float, so the moments decay with the fp32 betas
// (1 - 0.999f is 1.3e-5 below 0.001, so v is 1.3e-5 below torch's); the bias corrections use the same betas, which
// cancels that difference in the update.
#include "common.cuh"

namespace usip {

__global__ void __launch_bounds__(256)
adam_step_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
                 const float* __restrict__ lr_dev, long long* __restrict__ step_dev, unsigned int* __restrict__ arrive,
                 float beta1, float beta2, float eps, float grad_scale, long long n4) {
  const long long t = step_dev[0] + 1;
  const double bc1 = 1.0 - pow((double)beta1, (double)t), bc2 = 1.0 - pow((double)beta2, (double)t);
  const float step_size = (float)((double)lr_dev[0] / bc1);
  const float inv_bc2_sqrt = (float)(1.0 / sqrt(bc2));
  const float omb1 = 1.f - beta1, omb2 = 1.f - beta2;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    float4 g4 = reinterpret_cast<const float4*>(g)[i];
    float4 m4 = reinterpret_cast<float4*>(m)[i], v4 = reinterpret_cast<float4*>(v)[i], p4 = reinterpret_cast<float4*>(p)[i];
    float gv[4] = {g4.x * grad_scale, g4.y * grad_scale, g4.z * grad_scale, g4.w * grad_scale};
    float mv[4] = {m4.x, m4.y, m4.z, m4.w}, vv[4] = {v4.x, v4.y, v4.z, v4.w}, pv[4] = {p4.x, p4.y, p4.z, p4.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      mv[j] = __fadd_rn(__fmul_rn(mv[j], beta1), __fmul_rn(gv[j], omb1));                 // b1 m + (1-b1) g (not torch's lerp)
      vv[j] = __fadd_rn(__fmul_rn(vv[j], beta2), __fmul_rn(__fmul_rn(gv[j], gv[j]), omb2));
      const float denom = __fadd_rn(__fmul_rn(sqrtf(vv[j]), inv_bc2_sqrt), eps);
      pv[j] = __fsub_rn(pv[j], __fmul_rn(step_size, __fdiv_rn(mv[j], denom)));
    }
    reinterpret_cast<float4*>(m)[i] = make_float4(mv[0], mv[1], mv[2], mv[3]);
    reinterpret_cast<float4*>(v)[i] = make_float4(vv[0], vv[1], vv[2], vv[3]);
    reinterpret_cast<float4*>(p)[i] = make_float4(pv[0], pv[1], pv[2], pv[3]);
  }
  // every CTA has read step_dev before it arrives: the last one publishes the new step and re-arms the counter
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    if (atomicAdd(arrive, 1u) == gridDim.x - 1) { step_dev[0] = t; *arrive = 0u; __threadfence(); }
  }
}

}  // namespace usip

extern "C" int usip_adam_step(float* p, const float* g, float* m, float* v, const float* lr_dev, int64_t* step_dev,
                              uint32_t* arrive, float beta1, float beta2, float eps, float grad_scale, int64_t n,
                              void* stream) {
  using namespace usip;
  USIP_REQUIRE(n % 4 == 0, "adam_step: n must be a multiple of 4 (pad the flat buffer)");
  USIP_REQUIRE(((uintptr_t)p | (uintptr_t)g | (uintptr_t)m | (uintptr_t)v) % 16 == 0, "adam_step: 16-byte alignment");
  const long long n4 = n / 4;
  const long long want = cdiv64(n4, 256);
  const int blocks = (int)(want < device_sm_count() * 8 ? want : device_sm_count() * 8);
  adam_step_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(p, g, m, v, lr_dev, reinterpret_cast<long long*>(step_dev), arrive,
                                                             beta1, beta2, eps, grad_scale, n4);
  return check_launch("adam_step_kernel");
}
