// pairgen.cu -- device-side construction of the detector's training pairs (SURVEY section 8 f-2, completed): the random
// subsampling of data/kitti_detector_loader.py:118-145 (KittiLoader.get_instance_unaugmented_np), the augmentation of
// :149-216 (KittiLoader.augment) and the dst transform of data/augmentation.py:199-248 (transform_pc_pytorch).
//
// Randomness: per-pair scalars (angles, rotation matrices, scale, shifts) are drawn on the host and arrive as one
// `params` block per pair (usip_pair_augment).  Per-point randomness is either uploaded (the caller replays numpy's
// stream: the index lists and jitter arrays) or generated here with Philox4x32-10 keyed by (seed, step, cloud, point,
// purpose), so that a batch is a pure function of (seed, step).
//
// Clouds are numbered c = 2*pair + side (side 0 = src / anchor, 1 = dst / positive) and scan_of_cloud[c] names the scan
// cloud c is drawn from: the detector names every pair's scan twice (both sides subsample the same scan), the
// descriptor names the anchor's and the positive's.  The Philox counters depend on c only, so the mapping changes no
// random number.
#include "common.cuh"

namespace usip {

constexpr int PG_THREADS = 1024;                   // subset kernel: one CTA per cloud
constexpr int PG_AUG_THREADS = 256;
constexpr uint32_t PG_SENTINEL = 0xffffffffu;      // key of a point that may not be drawn (outside the radius)
constexpr int PG_PARAM_STRIDE = 48;                // doubles per pair, see usip_pair_augment in the header
constexpr int PG_DESC_PARAM_STRIDE = 32;           // doubles per cloud, see usip_desc_pair_augment in the header

enum { PURPOSE_ROWS = 0, PURPOSE_CAND = 1, PURPOSE_START = 2, PURPOSE_JIT_PC = 3, PURPOSE_JIT_SN = 4,
       PURPOSE_JIT_NODE = 5 };

// ---------------------------------------------------------------------------------------------- Philox4x32-10
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

__device__ __forceinline__ uint4 pg_random(uint64_t seed, uint64_t step, int cloud, int item, int purpose, int sub) {
  const uint4 ctr = make_uint4((uint32_t)item, (uint32_t)cloud, (uint32_t)step,
                               (uint32_t)purpose | ((uint32_t)sub << 8) | ((uint32_t)(step >> 32) << 16));
  return philox4x32_10(ctr, (uint32_t)seed, (uint32_t)(seed >> 32));
}

// two standard normals from two 32-bit words (Box-Muller in double, u1 in (0, 1])
__device__ __forceinline__ void pg_normal2(uint32_t a, uint32_t b, double& z0, double& z1) {
  const double u1 = ((double)a + 1.0) * 2.3283064365386963e-10;
  const double u2 = (double)b * 2.3283064365386963e-10;
  const double r = sqrt(-2.0 * log(u1));
  double s, c;
  sincospi(2.0 * u2, &s, &c);
  z0 = r * c; z1 = r * s;
}

__device__ __forceinline__ double pg_clip(double v, double lim) { return fmin(fmax(v, -lim), lim); }

// ------------------------------------------------------------------------------------------ block primitives
__device__ __forceinline__ uint64_t block_exclusive_scan_u64(uint64_t v, uint64_t* s_warp) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = blockDim.x >> 5;
  uint64_t inc = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint64_t t = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += t;
  }
  if (lane == 31) s_warp[w] = inc;
  __syncthreads();
  if (w == 0) {
    const uint64_t x = lane < nw ? s_warp[lane] : 0;
    uint64_t xi = x;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint64_t t = __shfl_up_sync(0xffffffffu, xi, o);
      if (lane >= o) xi += t;
    }
    s_warp[lane] = xi - x;
  }
  __syncthreads();
  const uint64_t r = s_warp[w] + inc - v;
  __syncthreads();
  return r;
}

// The `need` smallest (key, index) pairs among the keys != PG_SENTINEL: returns the threshold key T and how many of the
// keys equal to T are taken (the lowest indices).  Four 8-bit radix passes over shared memory.  1 <= need <= #eligible.
__device__ void pg_radix_threshold(const uint32_t* key, int n, int need, uint32_t* hist, uint32_t* s_ctl,
                                   uint32_t& T, int& take) {
  const int tid = threadIdx.x, lane = tid & 31;
  uint32_t prefix = 0, pmask = 0, rem = (uint32_t)need;
  for (int shift = 24; shift >= 0; shift -= 8) {
    for (int i = tid; i < 256; i += blockDim.x) hist[i] = 0;
    __syncthreads();
    for (int i = tid; i < n; i += blockDim.x) {
      const uint32_t k = key[i];
      if (k != PG_SENTINEL && (k & pmask) == prefix) atomicAdd(&hist[(k >> shift) & 255u], 1u);
    }
    __syncthreads();
    if (tid < 32) {
      uint32_t loc[8], s = 0;
#pragma unroll
      for (int j = 0; j < 8; ++j) { loc[j] = hist[lane * 8 + j]; s += loc[j]; }
      uint32_t inc = s;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const uint32_t t = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += t;
      }
      uint32_t c = inc - s;
      if (c < rem && rem <= inc) {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          if (c < rem && rem <= c + loc[j]) { s_ctl[0] = (uint32_t)(lane * 8 + j); s_ctl[1] = rem - c; }
          c += loc[j];
        }
      }
    }
    __syncthreads();
    prefix |= s_ctl[0] << shift;
    pmask |= 0xffu << shift;
    rem = s_ctl[1];
  }
  T = prefix; take = (int)rem;
}

// Radius mask of kitti_detector_loader.py:119-123: np.linalg.norm(pc[:, [0, 2]], axis=1) <= r, i.e. sqrt(x*x + z*z)
// in fp32 without contraction, compared in double.
__device__ __forceinline__ bool pg_inside(const float* p, double radius) {
  const float n = __fsqrt_rn(__fadd_rn(__fmul_rn(p[0], p[0]), __fmul_rn(p[2], p[2])));
  return (double)n <= radius;
}

// level 0: rows of every cloud (uniform subset of N without replacement, or the reference's "tile all, then a random
//          remainder" when fewer than N points survive the mask), ascending raw row index inside each part;
// level 1: the N/3 FPS candidates as ascending positions into the rows, and the FPS start index.
__global__ void __launch_bounds__(PG_THREADS)
pair_subset_kernel(const float* __restrict__ scans, int C, const int64_t* __restrict__ offsets,
                   const int32_t* __restrict__ scan_of_cloud, int level, int use_radius, double radius, int N,
                   int n_cand, uint64_t seed, uint64_t step, int32_t* __restrict__ out_rows,
                   int32_t* __restrict__ out_cand, int32_t* __restrict__ out_start, int32_t* __restrict__ out_valid) {
  extern __shared__ __align__(16) unsigned char pg_smem[];
  __shared__ uint32_t hist[256];
  __shared__ uint32_t s_ctl[2];
  __shared__ uint64_t s_warp[32];
  uint32_t* key = reinterpret_cast<uint32_t*>(pg_smem);
  const int c = blockIdx.x, tid = threadIdx.x;
  const int scan = scan_of_cloud[c];
  const int64_t row0 = offsets[scan];
  const int n = level == 0 ? (int)(offsets[scan + 1] - row0) : N;
  const float* base = scans + row0 * C;

  // keys: 31 random bits, so that no drawable point carries the sentinel
  int my_valid = 0;
  for (int i = tid; i < n; i += blockDim.x) {
    const bool ok = level != 0 || !use_radius || pg_inside(base + (int64_t)i * C, radius);
    key[i] = ok ? (pg_random(seed, step, c, i, level == 0 ? PURPOSE_ROWS : PURPOSE_CAND, 0).x >> 1) : PG_SENTINEL;
    my_valid += ok;
  }
  const uint64_t nvalid_excl = block_exclusive_scan_u64((uint64_t)my_valid, s_warp);
  if (tid == blockDim.x - 1) s_ctl[0] = (uint32_t)(nvalid_excl + my_valid);
  __syncthreads();
  const int nvalid = (int)s_ctl[0];
  __syncthreads();

  int tiles = 0, need = level == 0 ? N : n_cand;
  if (level == 0) {
    if (out_valid && tid == 0) out_valid[c] = nvalid;
    if (nvalid == 0) {                              // nothing to draw from: every row is 0 (see the header)
      for (int i = tid; i < N; i += blockDim.x) out_rows[(int64_t)c * N + i] = 0;
      return;
    }
    if (nvalid < N) {                               // kitti_detector_loader.py:129-133
      tiles = max(1, (N + nvalid - 1) / nvalid - 1);
      need = N - tiles * nvalid;
    }
  } else if (tid == 0) {
    const uint32_t r = pg_random(seed, step, c, 0, PURPOSE_START, 0).x;
    out_start[c] = (int32_t)(((uint64_t)r * (uint64_t)n_cand) >> 32);
  }

  uint32_t T = 0; int take = 0;
  if (need > 0) pg_radix_threshold(key, n, need, hist, s_ctl, T, take);

  // ordered emission: each thread owns a contiguous chunk, one block scan of (less, equal, valid) counts
  const int chunk = (n + blockDim.x - 1) / blockDim.x;
  const int i0 = min(n, tid * chunk), i1 = min(n, i0 + chunk);
  uint64_t cnt = 0;
  for (int i = i0; i < i1; ++i) {
    const uint32_t k = key[i];
    if (k == PG_SENTINEL) continue;
    cnt += (need > 0 && k < T) ? 1ull : 0ull;
    cnt += (need > 0 && k == T) ? (1ull << 21) : 0ull;
    cnt += 1ull << 42;
  }
  const uint64_t ex = block_exclusive_scan_u64(cnt, s_warp);
  int less = (int)(ex & 0x1fffff), eq = (int)((ex >> 21) & 0x1fffff), vr = (int)(ex >> 42);
  int32_t* out = level == 0 ? out_rows + (int64_t)c * N : out_cand + (int64_t)c * n_cand;
  const int sel_base = tiles * nvalid;
  for (int i = i0; i < i1; ++i) {
    const uint32_t k = key[i];
    if (k == PG_SENTINEL) continue;
    for (int t = 0; t < tiles; ++t) out[t * nvalid + vr] = i;
    if (need > 0) {
      if (k < T) out[sel_base + less + min(eq, take)] = i;
      else if (k == T && eq < take) out[sel_base + less + eq] = i;
      less += k < T;
      eq += k == T;
    }
    ++vr;
  }
}

// candidate points for FPS: pts[c, j, :] = xyz of row rows[c, cand[c, j]]
__global__ void pair_gather_kernel(const float* __restrict__ scans, int C, const int64_t* __restrict__ offsets,
                                   const int32_t* __restrict__ scan_of_cloud, const int32_t* __restrict__ rows,
                                   const int32_t* __restrict__ cand, float* __restrict__ pts, int N, int n_cand) {
  const int c = blockIdx.y, j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n_cand) return;
  const int r = rows[(int64_t)c * N + cand[(int64_t)c * n_cand + j]];
  const float* p = scans + (offsets[scan_of_cloud[c]] + r) * C;
  float* o = pts + ((int64_t)c * n_cand + j) * 3;
  o[0] = p[0]; o[1] = p[1]; o[2] = p[2];
}

// row vector times R (numpy `data @ R`, augmentation.py:62-72), float64.  The host BLAS (numpy's dgemm) accumulates
// k = 0, 1, 2 as a fused multiply-add chain started by a plain product; the same chain here reproduces its bits.
__device__ __forceinline__ void pg_rowvec(double& x, double& y, double& z, const double* R) {
  const double a = x, b = y, c = z;
  x = __fma_rn(c, R[6], __fma_rn(b, R[3], __dmul_rn(a, R[0])));
  y = __fma_rn(c, R[7], __fma_rn(b, R[4], __dmul_rn(a, R[1])));
  z = __fma_rn(c, R[8], __fma_rn(b, R[5], __dmul_rn(a, R[2])));
}

// R times column vector in fp32 (torch.matmul(R, pc), augmentation.py:231-235): the same k = 0, 1, 2 FMA chain as
// torch's CPU sgemm
__device__ __forceinline__ void pg_colvec(float& x, float& y, float& z, const float* R) {
  const float a = x, b = y, c = z;
  x = __fmaf_rn(R[2], c, __fmaf_rn(R[1], b, __fmul_rn(R[0], a)));
  y = __fmaf_rn(R[5], c, __fmaf_rn(R[4], b, __fmul_rn(R[3], a)));
  z = __fmaf_rn(R[8], c, __fmaf_rn(R[7], b, __fmul_rn(R[6], a)));
}

constexpr int PG_MAX_S = 8;

// --------------------------------------------------------------- train-time augmentation shared by both loaders
// kitti_detector_loader.py:182-212 (KittiLoader.augment) and kitti_descriptor_loader.py:240-272
// (KittiDescriptorLoader.augment) apply the same arithmetic to every cloud; these helpers are that arithmetic, so the
// two kernels cannot drift apart.  P points at one cloud's [0:27] rotation matrices (horizontal, 3-d, perturbation)
// and [28:31] shift; sc is the augmentation scale; flags the USIP_PAIR_* bits.
// Flags: USIP_PAIR_ROT_HORIZONTAL << r is rotation r.
constexpr int PG_ANY_ROT = USIP_PAIR_ROT_HORIZONTAL | USIP_PAIR_ROT_3D | USIP_PAIR_ROT_PERTURBATION;

// clipped N(0, 0.04^2) jitter of one point or node (pc and nodes use the same law): uploaded, or Philox
__device__ __forceinline__ void pg_jitter_xyz(const double* jit, int64_t at, uint64_t seed, uint64_t step, int c, int i,
                                              int purpose, double j[4]) {
  if (jit) {
    const double* q = jit + at * 3;
    j[0] = q[0]; j[1] = q[1]; j[2] = q[2];
  } else {
    const uint4 u = pg_random(seed, step, c, i, purpose, 0);
    pg_normal2(u.x, u.y, j[0], j[1]); pg_normal2(u.z, u.w, j[2], j[3]);
#pragma unroll
    for (int k = 0; k < 3; ++k) j[k] = pg_clip(0.04 * j[k], 0.12);
  }
}

// one point: rotations (pc in float64, sn a float32 view rounded after every rotation), jitter, scale, shift
__device__ __forceinline__ void pg_augment_point(int flags, const double* P, double sc, const double* j, int S,
                                                 float& x, float& y, float& z, float* sn) {
  double X = x, Y = y, Z = z;
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    if (!(flags & (USIP_PAIR_ROT_HORIZONTAL << r))) continue;
    pg_rowvec(X, Y, Z, P + 9 * r);
    if (S >= 3) {
      double a = sn[0], bb = sn[1], cc = sn[2];
      pg_rowvec(a, bb, cc, P + 9 * r);
      sn[0] = (float)a; sn[1] = (float)bb; sn[2] = (float)cc;
    }
  }
  if (flags & PG_ANY_ROT) {                                 // pc is float64 after the first rotation
    X = __dadd_rn(X, j[0]); Y = __dadd_rn(Y, j[1]); Z = __dadd_rn(Z, j[2]);
    X = __dmul_rn(X, sc); Y = __dmul_rn(Y, sc); Z = __dmul_rn(Z, sc);
    if (flags & USIP_PAIR_TRANSLATION) { X = __dadd_rn(X, P[28]); Y = __dadd_rn(Y, P[29]); Z = __dadd_rn(Z, P[30]); }
    x = (float)X; y = (float)Y; z = (float)Z;
  } else {                                         // pc is still the float32 slice: every step rounds to fp32
    x = (float)__dadd_rn((double)x, j[0]); y = (float)__dadd_rn((double)y, j[1]);
    z = (float)__dadd_rn((double)z, j[2]);
    const float scf = (float)sc;                   // float32 array * Python float
    x = __fmul_rn(x, scf); y = __fmul_rn(y, scf); z = __fmul_rn(z, scf);
    if (flags & USIP_PAIR_TRANSLATION) {
      x = (float)__dadd_rn((double)x, P[28]); y = (float)__dadd_rn((double)y, P[29]);
      z = (float)__dadd_rn((double)z, P[30]);
    }
  }
}

// sn jitter: fl32(double(sn) + j) with j clipped N(0, 0.01^2), never scaled or shifted; at = the point's row in jit_sn
__device__ __forceinline__ void pg_jitter_sn(const double* jit_sn, int64_t at, uint64_t seed, uint64_t step, int c,
                                             int i, int S, float* sn) {
#pragma unroll
  for (int q = 0; q < PG_MAX_S; q += 4) {
    if (q >= S) break;
    double js[4];
    if (jit_sn) {
#pragma unroll
      for (int k = 0; k < 4; ++k) js[k] = q + k < S ? jit_sn[at * S + q + k] : 0.0;
    } else {
      const uint4 u = pg_random(seed, step, c, i, PURPOSE_JIT_SN, q / 4);
      pg_normal2(u.x, u.y, js[0], js[1]); pg_normal2(u.z, u.w, js[2], js[3]);
#pragma unroll
      for (int k = 0; k < 4; ++k) js[k] = pg_clip(0.01 * js[k], 0.05);
    }
#pragma unroll
    for (int k = 0; k < 4; ++k)
      if (q + k < S) sn[q + k] = (float)__dadd_rn((double)sn[q + k], js[k]);
  }
}

// one node: float64 (FarthestSampler output) through rotations, jitter, scale and shift until the final cast
__device__ __forceinline__ void pg_augment_node(int flags, const double* P, double sc, const double* j, float& x,
                                                float& y, float& z) {
  double X = x, Y = y, Z = z;
#pragma unroll
  for (int r = 0; r < 3; ++r)
    if (flags & (USIP_PAIR_ROT_HORIZONTAL << r)) pg_rowvec(X, Y, Z, P + 9 * r);
  X = __dmul_rn(__dadd_rn(X, j[0]), sc); Y = __dmul_rn(__dadd_rn(Y, j[1]), sc); Z = __dmul_rn(__dadd_rn(Z, j[2]), sc);
  if (flags & USIP_PAIR_TRANSLATION) { X = __dadd_rn(X, P[28]); Y = __dadd_rn(Y, P[29]); Z = __dadd_rn(Z, P[30]); }
  x = (float)X; y = (float)Y; z = (float)Z;
}

__global__ void __launch_bounds__(PG_AUG_THREADS)
pair_augment_kernel(const float* __restrict__ scans, int C, const int64_t* __restrict__ offsets,
                    const int32_t* __restrict__ scan_of_cloud, const int32_t* __restrict__ rows,
                    const float* __restrict__ nodes, const double* __restrict__ params,
                    const double* __restrict__ jit_pc, const double* __restrict__ jit_sn,
                    const double* __restrict__ jit_node, uint64_t seed, uint64_t step, int flags, int S, int sn_col,
                    int N, int M, float* __restrict__ src_pc, float* __restrict__ src_sn, float* __restrict__ src_node,
                    float* __restrict__ dst_pc, float* __restrict__ dst_sn, float* __restrict__ dst_node,
                    float* __restrict__ R_out, float* __restrict__ scale_out, float* __restrict__ shift_out) {
  const int c = blockIdx.y, b = c >> 1, side = c & 1;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const double* P = params + (int64_t)b * PG_PARAM_STRIDE;
  const bool train = flags & USIP_PAIR_TRAIN;
  float RT[9];
#pragma unroll
  for (int k = 0; k < 9; ++k) RT[k] = (float)P[31 + k];

  if (side == 1 && blockIdx.x == 0) {
    if (threadIdx.x < 9) R_out[b * 9 + threadIdx.x] = RT[threadIdx.x];
    else if (threadIdx.x == 9) scale_out[b] = (float)P[43];
    else if (threadIdx.x < 13) shift_out[b * 3 + threadIdx.x - 10] = (float)P[40 + threadIdx.x - 10];
  }

  if (i < N) {
    const int64_t row = offsets[scan_of_cloud[c]] + rows[(int64_t)c * N + i];
    const float* p = scans + row * C;
    float x = p[0], y = p[1], z = p[2];
    float sn[PG_MAX_S];
#pragma unroll
    for (int k = 0; k < PG_MAX_S; ++k) sn[k] = k < S ? p[sn_col + k] : 0.f;
    if (train) {                                   // KittiLoader.augment, :182-212
      double j[4];
      pg_jitter_xyz(jit_pc, (int64_t)c * N + i, seed, step, c, i, PURPOSE_JIT_PC, j);
      pg_augment_point(flags, P, P[27], j, S, x, y, z, sn);
      pg_jitter_sn(jit_sn, (int64_t)c * N + i, seed, step, c, i, S, sn);
    }
    float* opc = side ? dst_pc : src_pc;
    float* osn = side ? dst_sn : src_sn;
    if (side == 1) {                               // transform_pc_pytorch, fp32, column vectors
      pg_colvec(x, y, z, RT);
      if (S >= 3) pg_colvec(sn[0], sn[1], sn[2], RT);
      const float sc = (float)P[43];
      x = __fmul_rn(x, sc); y = __fmul_rn(y, sc); z = __fmul_rn(z, sc);
      x = __fadd_rn(x, (float)P[40]); y = __fadd_rn(y, (float)P[41]); z = __fadd_rn(z, (float)P[42]);
    }
    opc[((int64_t)b * 3 + 0) * N + i] = x;
    opc[((int64_t)b * 3 + 1) * N + i] = y;
    opc[((int64_t)b * 3 + 2) * N + i] = z;
#pragma unroll
    for (int k = 0; k < PG_MAX_S; ++k)
      if (k < S) osn[((int64_t)b * S + k) * N + i] = sn[k];
  }

  if (i < M) {
    const float* nd = nodes + (int64_t)c * 3 * M;
    float x = nd[i], y = nd[M + i], z = nd[2 * M + i];
    if (train) {
      double j[4];
      pg_jitter_xyz(jit_node, (int64_t)c * M + i, seed, step, c, i, PURPOSE_JIT_NODE, j);
      pg_augment_node(flags, P, P[27], j, x, y, z);
    }
    float* ond = side ? dst_node : src_node;
    if (side == 1) {
      pg_colvec(x, y, z, RT);
      const float sc = (float)P[43];
      x = __fmul_rn(x, sc); y = __fmul_rn(y, sc); z = __fmul_rn(z, sc);
      x = __fadd_rn(x, (float)P[40]); y = __fadd_rn(y, (float)P[41]); z = __fadd_rn(z, (float)P[42]);
    }
    ond[((int64_t)b * 3 + 0) * M + i] = x;
    ond[((int64_t)b * 3 + 1) * M + i] = y;
    ond[((int64_t)b * 3 + 2) * M + i] = z;
  }
}

// Descriptor pairs (KittiDescriptorLoader.augment, kitti_descriptor_loader.py:205-276): every cloud has its own scan,
// rotations, jitter and shift; the scale is the pair's, in both clouds' [27].  No dst transform.  sn = columns 3:3+S
// for every S.
__global__ void __launch_bounds__(PG_AUG_THREADS)
desc_pair_augment_kernel(const float* __restrict__ scans, int C, const int64_t* __restrict__ offsets,
                         const int32_t* __restrict__ scan_of_cloud, const int32_t* __restrict__ rows,
                         const float* __restrict__ nodes, const double* __restrict__ params,
                         const double* __restrict__ jit_pc, const double* __restrict__ jit_sn,
                         const double* __restrict__ jit_node, uint64_t seed, uint64_t step, int flags, int S, int N,
                         int M, float* __restrict__ anc_pc, float* __restrict__ anc_sn, float* __restrict__ anc_node,
                         float* __restrict__ pos_pc, float* __restrict__ pos_sn, float* __restrict__ pos_node) {
  const int c = blockIdx.y, b = c >> 1, side = c & 1;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const double* P = params + (int64_t)c * PG_DESC_PARAM_STRIDE;
  const bool train = flags & USIP_PAIR_TRAIN;

  if (i < N) {
    const float* p = scans + (offsets[scan_of_cloud[c]] + rows[(int64_t)c * N + i]) * C;
    float x = p[0], y = p[1], z = p[2];
    float sn[PG_MAX_S];
#pragma unroll
    for (int k = 0; k < PG_MAX_S; ++k) sn[k] = k < S ? p[3 + k] : 0.f;
    if (train) {
      double j[4];
      pg_jitter_xyz(jit_pc, (int64_t)c * N + i, seed, step, c, i, PURPOSE_JIT_PC, j);
      pg_augment_point(flags, P, P[27], j, S, x, y, z, sn);
      pg_jitter_sn(jit_sn, (int64_t)c * N + i, seed, step, c, i, S, sn);
    }
    float* opc = side ? pos_pc : anc_pc;
    float* osn = side ? pos_sn : anc_sn;
    opc[((int64_t)b * 3 + 0) * N + i] = x;
    opc[((int64_t)b * 3 + 1) * N + i] = y;
    opc[((int64_t)b * 3 + 2) * N + i] = z;
#pragma unroll
    for (int k = 0; k < PG_MAX_S; ++k)
      if (k < S) osn[((int64_t)b * S + k) * N + i] = sn[k];
  }

  if (i < M) {
    const float* nd = nodes + (int64_t)c * 3 * M;
    float x = nd[i], y = nd[M + i], z = nd[2 * M + i];
    if (train) {
      double j[4];
      pg_jitter_xyz(jit_node, (int64_t)c * M + i, seed, step, c, i, PURPOSE_JIT_NODE, j);
      pg_augment_node(flags, P, P[27], j, x, y, z);
    }
    float* ond = side ? pos_node : anc_node;
    ond[((int64_t)b * 3 + 0) * M + i] = x;
    ond[((int64_t)b * 3 + 1) * M + i] = y;
    ond[((int64_t)b * 3 + 2) * M + i] = z;
  }
}

}  // namespace usip

using namespace usip;

static int pg_subset_smem(int n) { return n * (int)sizeof(uint32_t); }

extern "C" int usip_pair_max_scan_rows(void) {
  return (227 * 1024 - 4096) / (int)sizeof(uint32_t);
}

// rows, then candidates + FPS start, of 2*n_pairs clouds
extern "C" int usip_cloud_subsample(const float* scans, int C, const int64_t* offsets, const int32_t* scan_of_cloud,
                                    int max_rows, int n_pairs, int N, int n_cand, int use_radius, double radius,
                                    uint64_t seed, uint64_t step, int32_t* out_rows, int32_t* out_cand,
                                    int32_t* out_start, int32_t* out_valid, void* stream) {
  USIP_REQUIRE(scans && offsets && scan_of_cloud && out_rows && out_cand && out_start, "cloud_subsample: null pointer");
  USIP_REQUIRE(C >= 3 && n_pairs > 0 && N > 0 && n_cand > 0 && n_cand <= N && max_rows > 0,
               "cloud_subsample: bad sizes");
  USIP_REQUIRE(max(max_rows, N) <= usip_pair_max_scan_rows(),
               "cloud_subsample: scan or N too large for shared memory");
  cudaError_t e = cudaFuncSetAttribute(pair_subset_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       pg_subset_smem(max(max_rows, N)));
  if (e != cudaSuccess) { set_last_error("cloud_subsample: smem attribute"); return (int)e; }
  cudaStream_t s = (cudaStream_t)stream;
  pair_subset_kernel<<<2 * n_pairs, PG_THREADS, pg_subset_smem(max_rows), s>>>(
      scans, C, offsets, scan_of_cloud, 0, use_radius, radius, N, n_cand, seed, step, out_rows, out_cand, out_start,
      out_valid);
  int rc = check_launch("pair_subset_kernel(rows)");
  if (rc) return rc;
  pair_subset_kernel<<<2 * n_pairs, PG_THREADS, pg_subset_smem(N), s>>>(
      scans, C, offsets, scan_of_cloud, 1, 0, 0.0, N, n_cand, seed, step, out_rows, out_cand, out_start, out_valid);
  return check_launch("pair_subset_kernel(candidates)");
}

extern "C" int usip_cloud_gather_candidates(const float* scans, int C, const int64_t* offsets,
                                            const int32_t* scan_of_cloud, const int32_t* rows, const int32_t* cand,
                                            float* out_pts, int n_pairs, int N, int n_cand, void* stream) {
  USIP_REQUIRE(scans && offsets && scan_of_cloud && rows && cand && out_pts, "cloud_gather_candidates: null pointer");
  USIP_REQUIRE(C >= 3 && n_pairs > 0 && N > 0 && n_cand > 0 && n_cand <= N, "cloud_gather_candidates: bad sizes");
  dim3 grid(cdiv(n_cand, 256), 2 * n_pairs);
  pair_gather_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(scans, C, offsets, scan_of_cloud, rows, cand, out_pts, N,
                                                              n_cand);
  return check_launch("pair_gather_kernel");
}

extern "C" int usip_desc_pair_augment(const float* scans, int C, const int64_t* offsets, const int32_t* scan_of_cloud,
                                      const int32_t* rows, const float* nodes, const double* params,
                                      const double* jit_pc, const double* jit_sn, const double* jit_node,
                                      uint64_t seed, uint64_t step, int flags, int S, int n_pairs, int N, int M,
                                      float* anc_pc, float* anc_sn, float* anc_node, float* pos_pc, float* pos_sn,
                                      float* pos_node, void* stream) {
  USIP_REQUIRE(scans && offsets && scan_of_cloud && rows && nodes && params, "desc_pair_augment: null input");
  USIP_REQUIRE(anc_pc && anc_sn && anc_node && pos_pc && pos_sn && pos_node, "desc_pair_augment: null output");
  USIP_REQUIRE(S >= 1 && S <= PG_MAX_S && 3 + S <= C, "desc_pair_augment: bad surface-normal length");
  USIP_REQUIRE(n_pairs > 0 && N > 0 && M > 0, "desc_pair_augment: bad sizes");
  dim3 grid(cdiv(max(N, M), PG_AUG_THREADS), 2 * n_pairs);
  desc_pair_augment_kernel<<<grid, PG_AUG_THREADS, 0, (cudaStream_t)stream>>>(
      scans, C, offsets, scan_of_cloud, rows, nodes, params, jit_pc, jit_sn, jit_node, seed, step, flags, S, N, M,
      anc_pc, anc_sn, anc_node, pos_pc, pos_sn, pos_node);
  return check_launch("desc_pair_augment_kernel");
}

extern "C" int usip_pair_augment(const float* scans, int C, const int64_t* offsets, const int32_t* scan_of_cloud,
                                 const int32_t* rows, const float* nodes, const double* params, const double* jit_pc,
                                 const double* jit_sn, const double* jit_node, uint64_t seed, uint64_t step, int flags,
                                 int S, int n_pairs, int N, int M, float* src_pc, float* src_sn, float* src_node,
                                 float* dst_pc, float* dst_sn, float* dst_node, float* R, float* scale, float* shift,
                                 void* stream) {
  USIP_REQUIRE(scans && offsets && scan_of_cloud && rows && nodes && params, "pair_augment: null input");
  USIP_REQUIRE(src_pc && src_sn && src_node && dst_pc && dst_sn && dst_node && R && scale && shift,
               "pair_augment: null output");
  USIP_REQUIRE(S >= 1 && S <= PG_MAX_S && (S == 1 || 3 + S <= C) && C >= 4, "pair_augment: bad surface-normal length");
  USIP_REQUIRE(n_pairs > 0 && N > 0 && M > 0, "pair_augment: bad sizes");
  const int sn_col = S == 1 ? C - 1 : 3;           // kitti_detector_loader.py:135-139
  dim3 grid(cdiv(max(N, M), PG_AUG_THREADS), 2 * n_pairs);
  pair_augment_kernel<<<grid, PG_AUG_THREADS, 0, (cudaStream_t)stream>>>(
      scans, C, offsets, scan_of_cloud, rows, nodes, params, jit_pc, jit_sn, jit_node, seed, step, flags, S, sn_col, N,
      M, src_pc, src_sn, src_node, dst_pc, dst_sn, dst_node, R, scale, shift);
  return check_launch("pair_augment_kernel");
}
