// tc_common.cuh -- PTX wrappers shared by the Hopper tensor-core kernels (mbarrier, TMA bulk copy, wgmma descriptors) and
// the host-side tensor-map encoder.
#pragma once
#include "common.cuh"
#include <cuda.h>           // CUtensorMap types only; the encoder is resolved at run time

namespace usip {

constexpr int TC_BM = 128;                 // rows per CTA tile: two warpgroups, one m64 wgmma row block each
constexpr int TC_WG_ROWS = 64;             // rows per warpgroup tile of the layer kernel (one m64 wgmma row block)
constexpr int TC_BK = 32;                  // floats per K chunk (= one 128-byte swizzle row)

// ------------------------------------------------------------------------------------------------ PTX
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_LOOP:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra WAIT_DONE;\n"
      "bra WAIT_LOOP;\n"
      "WAIT_DONE:\n"
      "}\n" ::"r"(bar), "r"(parity)
      : "memory");
}
// wait with a suspend-time hint: the warp sleeps in hardware until the phase completes (or ~2 us pass) instead of spinning
// on try_wait -- for kernels where MANY warps wait on their own barrier and a spin would eat the issue slots of the others
__device__ __forceinline__ void mbar_wait_sleep(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAITS_LOOP:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1, %2;\n"
      "@p bra WAITS_DONE;\n"
      "bra WAITS_LOOP;\n"
      "WAITS_DONE:\n"
      "}\n" ::"r"(bar), "r"(parity), "r"(2000u)
      : "memory");
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
// per-thread register budget of the executing warpgroup (all its warps execute it): hands registers from a producer
// warpgroup to the consumers
template <int R> __device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R> __device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }
// barrier `id` (1..15; 0 is __syncthreads) over `threads` threads, a multiple of 32: couples only the warps that use it
__device__ __forceinline__ void named_bar_sync(int id, int threads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ void bulk_g2s(uint32_t dst_smem, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst_smem),
               "l"(src), "r"(bytes), "r"(bar)
               : "memory");
}
// box {c0.., c1..} of a 2-D tensor map (a __grid_constant__ parameter) -> shared memory.  Elements past the tensor's
// bounds arrive as zeros, and the barrier's transaction still counts the whole box.
__device__ __forceinline__ void tma_load_2d(uint32_t dst_smem, const CUtensorMap* map, int c0, int c1, uint32_t bar) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
               ::"r"(dst_smem), "l"(map), "r"(c0), "r"(c1), "r"(bar)
               : "memory");
}
__device__ __forceinline__ void prefetch_tensor_map(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(map) : "memory");
}

// cuTensorMapEncodeTiled (no interleave, out-of-bounds elements read as zeros), resolved once through the runtime
// (cudaGetDriverEntryPoint): the library keeps no link-time dependency on libcuda, so it still loads (and exports its
// symbols) on a machine without a driver.  Returns 0, or an error code with the last error set to `what`.
inline int encode_tensor_map_tiled(CUtensorMap* tm, CUtensorMapDataType dtype, cuuint32_t rank, void* gaddr,
                                   const cuuint64_t* dims, const cuuint64_t* strides, const cuuint32_t* box,
                                   const cuuint32_t* estr, CUtensorMapSwizzle swizzle, CUtensorMapL2promotion l2,
                                   const char* what) {
  typedef CUresult (*EncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                               const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                               CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
  static EncodeFn encode = nullptr;
  if (!encode) {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres);
    if (e != cudaSuccess || !fn) { set_last_error(what); return e != cudaSuccess ? (int)e : -1; }
    encode = (EncodeFn)fn;
  }
  CUresult r = encode(tm, dtype, rank, gaddr, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle, l2,
                      CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_last_error(what); return (int)r; }
  return 0;
}

__device__ __forceinline__ uint32_t to_tf32(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return r;
}
__device__ __forceinline__ void split_tf32(float x, uint32_t& hi, uint32_t& lo) {
  hi = to_tf32(x);
  lo = to_tf32(x - __uint_as_float(hi));
}

// ------------------------------------------------------------------------------------------------ wgmma (sm_90a)
// Operand tiles are K-major, SWIZZLE_128B: row r (128 B = 32 tf32) at r*128, 16-byte chunk c stored at chunk (c ^ (r & 7));
// 8-row groups 1024 B apart.  Tiles must start 1024-B aligned.  Descriptor (PTX "matrix descriptor", sm_90):
//  [0,14) start>>4 | [16,30) LBO>>4 (unused for swizzled K-major: 1) | [32,46) SBO>>4 (1024 B) | [62,64) layout 1 = 128B swizzle
// The k-th group of 8 tf32 inside the 128-byte row is addressed by advancing the start address by 32*k bytes.
__device__ __forceinline__ uint64_t make_kmajor_sw128_desc(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3FFFF) >> 4);
  d |= (uint64_t)1 << 16;
  d |= (uint64_t)(1024 >> 4) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accesses of the accumulator registers across a wgmma fence / wait
template <int R>
__device__ __forceinline__ void wgmma_fence_acc(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// D[64 x N] (+)= A[64 x 8] * B[N x 8]^T, tf32 operands from shared memory, fp32 accumulators in registers.
// Accumulator layout (per warp w of the warpgroup, lane l): d[4j + 0/1] = row 16w + l/4, columns 8j + 2(l%4) + 0/1;
// d[4j + 2/3] = the same columns of row 16w + l/4 + 8.
__device__ __forceinline__ void wgmma_tf32_n64(float (&d)[32], uint64_t adesc, uint64_t bdesc, uint32_t accum) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "setp.ne.b32 p, %34, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
      "%32, %33, p, 1, 1;\n"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(adesc), "l"(bdesc), "r"(accum)
      : "memory");
}
__device__ __forceinline__ void wgmma_tf32_n128(float (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t accum) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "setp.ne.b32 p, %66, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "%64, %65, p, 1, 1;\n"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(adesc), "l"(bdesc), "r"(accum)
      : "memory");
}

template <int BN>
__device__ __forceinline__ void wgmma_tf32(float (&d)[BN / 2], uint64_t adesc, uint64_t bdesc, uint32_t accum) {
  static_assert(BN == 64 || BN == 128, "wgmma tile width");
  if constexpr (BN == 64) wgmma_tf32_n64(d, adesc, bdesc, accum);
  else wgmma_tf32_n128(d, adesc, bdesc, accum);
}

// One 32-float K chunk of the warpgroup's [64 x BN] product, error-compensated 3xTF32 with a = a_hi + a_lo, b = b_hi + b_lo:
//     D += a_lo*b_hi + a_hi*b_lo + a_hi*b_hi        (dropped term a_lo*b_lo ~ 2^-22 relative)
// or, with SINGLE, plain TF32 (a_hi*b_hi only).  a_* point at this warpgroup's 64 operand rows, b_* at the BN rows of B.
// `first` zeroes the accumulator.  Issues one commit group; the caller waits on it.
template <int BN, bool SINGLE>
__device__ __forceinline__ void wgmma_chunk(float (&d)[BN / 2], uint32_t a_hi, uint32_t a_lo, uint32_t b_hi, uint32_t b_lo,
                                            bool first) {
  wgmma_fence_acc(d);
  wgmma_fence();
#pragma unroll
  for (int ks = 0; ks < TC_BK / 8; ++ks) {
    const uint64_t dah = make_kmajor_sw128_desc(a_hi + ks * 32), dbh = make_kmajor_sw128_desc(b_hi + ks * 32);
    const uint32_t acc = (first && ks == 0) ? 0u : 1u;
    if constexpr (SINGLE) {
      wgmma_tf32<BN>(d, dah, dbh, acc);
    } else {
      wgmma_tf32<BN>(d, make_kmajor_sw128_desc(a_lo + ks * 32), dbh, acc);
      wgmma_tf32<BN>(d, dah, make_kmajor_sw128_desc(b_lo + ks * 32), 1u);
      wgmma_tf32<BN>(d, dah, dbh, 1u);
    }
  }
  wgmma_commit();
  wgmma_fence_acc(d);
}

// D[64 x N] (+)= A[64 x 8] * B[N x 8]^T with A in registers (B as above).  A fragment of lane l of warp w of the warpgroup:
// a[0] = (row 16w + l/4, k l%4), a[1] = (row 16w + l/4 + 8, k l%4), a[2] = (row 16w + l/4, k l%4 + 4),
// a[3] = (row 16w + l/4 + 8, k l%4 + 4).  The registers must not change until the wgmma group that reads them retired.
__device__ __forceinline__ void wgmma_tf32_rs_n64(float (&d)[32], const uint32_t* a, uint64_t bdesc, uint32_t accum) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "setp.ne.b32 p, %37, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
      "{%32, %33, %34, %35}, %36, p, 1, 1;\n"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(accum)
      : "memory");
}
__device__ __forceinline__ void wgmma_tf32_rs_n128(float (&d)[64], const uint32_t* a, uint64_t bdesc, uint32_t accum) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "setp.ne.b32 p, %69, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "{%64, %65, %66, %67}, %68, p, 1, 1;\n"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(accum)
      : "memory");
}

// wgmma_chunk with the warpgroup's A fragments in registers: a_*[4ks .. 4ks+3] is the fragment of k-step ks.  b_hi points
// at the stage's [b_hi | b_lo] tile.  With SINGLE, a_lo is not read.
template <int BN, bool SINGLE>
__device__ __forceinline__ void wgmma_chunk_rs(float (&d)[BN / 2], const uint32_t (&a_hi)[16], const uint32_t (&a_lo)[16],
                                               uint32_t b_hi, bool first) {
  static_assert(BN == 64 || BN == 128, "wgmma tile width");
  const uint32_t b_lo = b_hi + BN * 128;
  wgmma_fence_acc(d);
  wgmma_fence();
#pragma unroll
  for (int ks = 0; ks < TC_BK / 8; ++ks) {
    const uint64_t dbh = make_kmajor_sw128_desc(b_hi + ks * 32);
    const uint32_t acc = (first && ks == 0) ? 0u : 1u;
    auto mma = [&](const uint32_t* a, uint64_t bdesc, uint32_t scale_d) {
      if constexpr (BN == 64) wgmma_tf32_rs_n64(d, a, bdesc, scale_d);
      else wgmma_tf32_rs_n128(d, a, bdesc, scale_d);
    };
    if constexpr (SINGLE) {
      mma(a_hi + 4 * ks, dbh, acc);
    } else {
      mma(a_lo + 4 * ks, dbh, acc);
      mma(a_hi + 4 * ks, make_kmajor_sw128_desc(b_lo + ks * 32), 1u);
      mma(a_hi + 4 * ks, dbh, 1u);
    }
  }
  wgmma_commit();
  wgmma_fence_acc(d);
}

}  // namespace usip
