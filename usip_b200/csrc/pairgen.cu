// pairgen.cu -- device-side construction of the detector's training pairs (SURVEY section 8 f-2, completed): the random
// subsampling of data/kitti_detector_loader.py:118-145 (KittiLoader.get_instance_unaugmented_np), the augmentation of
// :149-216 (KittiLoader.augment) and the dst transform of data/augmentation.py:199-248 (transform_pc_pytorch); the
// augmentation of data/modelnet_shrec_loader.py:182-243 (ModelNet_Shrec_Loader.augment, usip_modelnet_pair_augment);
// the ENU-to-camera frame and height scaling of the Oxford loaders (pg_enu_to_cam, usip_scale_channel_f32).
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
#include <cooperative_groups.h>

#include "common.cuh"

namespace cg = cooperative_groups;

namespace usip {

constexpr int PG_THREADS = 1024;                   // subset kernel: one CTA per cloud
constexpr int PG_AUG_THREADS = 256;
constexpr uint32_t PG_SENTINEL = 0xffffffffu;      // key of a point that may not be drawn (outside the radius)
constexpr int PG_PARAM_STRIDE = 48;                // doubles per pair, see usip_pair_augment in the header
constexpr int PG_AUGMENT_SLOT = 45;                // usip_indoor_pair_augment: params[b, 45] != 0 augments pair b
constexpr int PG_DESC_PARAM_STRIDE = 32;           // doubles per cloud, see usip_desc_pair_augment in the header
constexpr int PG_MAX_PAIRS = 32767;                // 2*n_pairs clouds run in grid.y, at most 65535

enum { PURPOSE_ROWS = 0, PURPOSE_CAND = 1, PURPOSE_START = 2, PURPOSE_JIT_PC = 3, PURPOSE_JIT_SN = 4,
       PURPOSE_JIT_NODE = 5, PURPOSE_NOISE = 6 };

// ---------------------------------------------------------------------------------------------- Philox4x32-10
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

// The subset's sort key of point i of cloud c: 31 random bits, so that no drawable point carries the sentinel, or
// PG_SENTINEL when the point may not be drawn.  Both subset kernels draw through this one expression.
__device__ __forceinline__ uint32_t pg_subset_key(bool ok, uint64_t seed, uint64_t step, int c, int i, int purpose) {
  return ok ? (pg_random(seed, step, c, i, purpose, 0).x >> 1) : PG_SENTINEL;
}

// One radix digit: warp 0 finds the bin of hist[256] that holds the rem-th smallest key and writes it to s_ctl[0] and
// the rank inside that bin to s_ctl[1].  The caller synchronises before reading s_ctl.
__device__ __forceinline__ void pg_radix_pick(const uint32_t* hist, uint32_t rem, uint32_t* s_ctl) {
  const int lane = threadIdx.x & 31;
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

// The `need` smallest (key, index) pairs among the keys != PG_SENTINEL: returns the threshold key T and how many of the
// keys equal to T are taken (the lowest indices).  Four 8-bit radix passes over shared memory.  1 <= need <= #eligible.
__device__ void pg_radix_threshold(const uint32_t* key, int n, int need, uint32_t* hist, uint32_t* s_ctl,
                                   uint32_t& T, int& take) {
  const int tid = threadIdx.x;
  uint32_t prefix = 0, pmask = 0, rem = (uint32_t)need;
  for (int shift = 24; shift >= 0; shift -= 8) {
    for (int i = tid; i < 256; i += blockDim.x) hist[i] = 0;
    __syncthreads();
    for (int i = tid; i < n; i += blockDim.x) {
      const uint32_t k = key[i];
      if (k != PG_SENTINEL && (k & pmask) == prefix) atomicAdd(&hist[(k >> shift) & 255u], 1u);
    }
    __syncthreads();
    if (tid < 32) pg_radix_pick(hist, rem, s_ctl);
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

  int my_valid = 0;
  for (int i = tid; i < n; i += blockDim.x) {
    const bool ok = level != 0 || !use_radius || pg_inside(base + (int64_t)i * C, radius);
    key[i] = pg_subset_key(ok, seed, step, c, i, level == 0 ? PURPOSE_ROWS : PURPOSE_CAND);
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

// Level 0 of a batch whose longest scan exceeds what pair_subset_kernel keeps in shared memory: one thread-block
// cluster of PG_CLUSTER CTAs per cloud, CTA r owning the contiguous slice [r*per, (r+1)*per) of the scan's rows.  No
// key is stored: every pass regenerates it with pg_subset_key, so the rows (the N smallest (key, row) pairs, the tile
// path, rows 0 without a valid point) and out_valid are exactly pair_subset_kernel's for the same (seed, step, cloud).
// The CTAs exchange their counts and radix histograms through distributed shared memory.  A slice has at most
// USIP_SUBSAMPLE_MAX_ROWS / PG_CLUSTER = 2^21 rows, so the counts are kept in 32 bits.
constexpr int PG_CLUSTER = 8;                      // the portable cluster size

__global__ void __cluster_dims__(PG_CLUSTER, 1, 1) __launch_bounds__(PG_THREADS)
pair_subset_cluster_kernel(const float* __restrict__ scans, int C, const int64_t* __restrict__ offsets,
                           const int32_t* __restrict__ scan_of_cloud, int use_radius, double radius, int N,
                           uint64_t seed, uint64_t step, int32_t* __restrict__ out_rows,
                           int32_t* __restrict__ out_valid) {
  cg::cluster_group cluster = cg::this_cluster();
  __shared__ uint32_t hist[256];
  __shared__ uint32_t s_ctl[2];
  __shared__ uint32_t s_part[3];                   // this CTA's (valid, less, equal) counts, read by the others
  __shared__ uint64_t s_warp[32];
  const int rank = (int)cluster.block_rank(), c = blockIdx.x / PG_CLUSTER, tid = threadIdx.x;
  const int scan = scan_of_cloud[c];
  const int64_t row0 = offsets[scan];
  const int n = (int)(offsets[scan + 1] - row0);
  const float* base = scans + row0 * C;
  const int per = (n + PG_CLUSTER - 1) / PG_CLUSTER;
  const int lo = min(n, rank * per), hi = min(n, lo + per);
  auto inside = [&](int i) { return !use_radius || pg_inside(base + (int64_t)i * C, radius); };
  auto key_of = [&](int i) { return pg_subset_key(inside(i), seed, step, c, i, PURPOSE_ROWS); };

  // pass 1: valid rows, in the whole scan and below this slice
  uint32_t my_valid = 0;
  for (int i = lo + tid; i < hi; i += blockDim.x) my_valid += inside(i);
  const uint64_t vex = block_exclusive_scan_u64(my_valid, s_warp);
  if (tid == blockDim.x - 1) s_part[0] = (uint32_t)(vex + my_valid);
  cluster.sync();
  int nvalid = 0, valid_base = 0;
  for (int r = 0; r < PG_CLUSTER; ++r) {
    const int v = (int)*cluster.map_shared_rank(&s_part[0], r);
    nvalid += v;
    valid_base += r < rank ? v : 0;
  }

  int tiles = 0, need = N;
  if (out_valid && rank == 0 && tid == 0) out_valid[c] = nvalid;
  if (nvalid == 0) {                               // nothing to draw from: every row is 0 (see the header)
    need = 0;
    for (int i = rank * blockDim.x + tid; i < N; i += PG_CLUSTER * blockDim.x) out_rows[(int64_t)c * N + i] = 0;
  } else if (nvalid < N) {                         // kitti_detector_loader.py:129-133
    tiles = max(1, (N + nvalid - 1) / nvalid - 1);
    need = N - tiles * nvalid;
  }

  // pass 2: four 8-bit radix passes; every CTA sums the eight histograms in rank order and picks the same digit
  uint32_t prefix = 0, pmask = 0, rem = (uint32_t)need;
  if (need > 0) {
    for (int shift = 24; shift >= 0; shift -= 8) {
      for (int i = tid; i < 256; i += blockDim.x) hist[i] = 0;
      __syncthreads();
      for (int i = lo + tid; i < hi; i += blockDim.x) {
        const uint32_t k = key_of(i);
        if (k != PG_SENTINEL && (k & pmask) == prefix) atomicAdd(&hist[(k >> shift) & 255u], 1u);
      }
      cluster.sync();                              // every slice's histogram is complete
      uint32_t sum = 0;
      if (tid < 256)
        for (int r = 0; r < PG_CLUSTER; ++r) sum += cluster.map_shared_rank(hist, r)[tid];
      cluster.sync();                              // no CTA clears its histogram while another still reads it
      if (tid < 256) hist[tid] = sum;
      __syncthreads();
      if (tid < 32) pg_radix_pick(hist, rem, s_ctl);
      __syncthreads();
      prefix |= s_ctl[0] << shift;
      pmask |= 0xffu << shift;
      rem = s_ctl[1];
    }
  }
  const uint32_t T = prefix;
  const int take = (int)rem;

  // pass 3: ordered emission.  Inside the CTA each thread owns a contiguous chunk of the slice (block scans of the
  // (less, equal) and valid counts); the CTA's base is the sum over the lower ranks.
  const int len = hi - lo, chunk = (len + blockDim.x - 1) / blockDim.x;
  const int i0 = lo + min(len, tid * chunk), i1 = lo + min(len, tid * chunk + chunk);
  uint64_t lt_eq = 0;
  uint32_t nv = 0;
  for (int i = i0; i < i1; ++i) {
    const uint32_t k = key_of(i);
    if (k == PG_SENTINEL) continue;
    lt_eq += (need > 0 && k < T) ? 1ull : 0ull;
    lt_eq += (need > 0 && k == T) ? (1ull << 32) : 0ull;
    ++nv;
  }
  const uint64_t ex = block_exclusive_scan_u64(lt_eq, s_warp);
  const uint64_t ex_v = block_exclusive_scan_u64(nv, s_warp);
  if (tid == blockDim.x - 1) {
    s_part[1] = (uint32_t)(ex + lt_eq);
    s_part[2] = (uint32_t)((ex + lt_eq) >> 32);
  }
  cluster.sync();
  int less = (int)(uint32_t)ex, eq = (int)(ex >> 32), vr = valid_base + (int)ex_v;
  for (int r = 0; r < rank; ++r) {
    less += (int)*cluster.map_shared_rank(&s_part[1], r);
    eq += (int)*cluster.map_shared_rank(&s_part[2], r);
  }
  int32_t* out = out_rows + (int64_t)c * N;
  const int sel_base = tiles * nvalid;
  for (int i = i0; i < i1; ++i) {
    const uint32_t k = key_of(i);
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
  cluster.sync();                                  // no CTA exits while another may still read its shared memory
}

// candidate points for FPS: pts[c, j, :] = xyz of row rows[c, cand[c, j]]; with z_scale, z is fl32(z * z_scale[c])
// (the Oxford detector's height scaling, which comes before its FPS)
__global__ void pair_gather_kernel(const float* __restrict__ scans, int C, const int64_t* __restrict__ offsets,
                                   const int32_t* __restrict__ scan_of_cloud, const int32_t* __restrict__ rows,
                                   const int32_t* __restrict__ cand, const float* __restrict__ z_scale,
                                   float* __restrict__ pts, int N, int n_cand) {
  const int c = blockIdx.y, j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n_cand) return;
  const int r = rows[(int64_t)c * N + cand[(int64_t)c * n_cand + j]];
  const float* p = scans + (offsets[scan_of_cloud[c]] + r) * C;
  float* o = pts + ((int64_t)c * n_cand + j) * 3;
  o[0] = p[0]; o[1] = p[1]; o[2] = z_scale ? __fmul_rn(p[2], z_scale[c]) : p[2];
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

// N(0, sigma^2) jitter clipped at +-clip of one point, normal or node: uploaded (row `at` of jit), or Philox keyed by
// (c, i, purpose).  The KITTI loaders jitter pc and nodes with sigma 0.04, clip 0.12; ModelNet's laws differ.
__device__ __forceinline__ void pg_jitter_xyz(const double* jit, int64_t at, uint64_t seed, uint64_t step, int c, int i,
                                              int purpose, double sigma, double clip, double j[4]) {
  if (jit) {
    const double* q = jit + at * 3;
    j[0] = q[0]; j[1] = q[1]; j[2] = q[2];
  } else {
    const uint4 u = pg_random(seed, step, c, i, purpose, 0);
    pg_normal2(u.x, u.y, j[0], j[1]); pg_normal2(u.z, u.w, j[2], j[3]);
#pragma unroll
    for (int k = 0; k < 3; ++k) j[k] = pg_clip(sigma * j[k], clip);
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

// sn jitter: fl32(double(sn) + j) with j clipped N(0, sigma^2), never scaled or shifted; at = the point's row in jit_sn
__device__ __forceinline__ void pg_jitter_sn(const double* jit_sn, int64_t at, uint64_t seed, uint64_t step, int c,
                                             int i, int S, double sigma, double clip, float* sn) {
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
      for (int k = 0; k < 4; ++k) js[k] = pg_clip(sigma * js[k], clip);
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

// The Oxford loaders' scans are ENU (z up).  coordinate_ENU_to_cam (augmentation.py:266-278) maps (x, y, z) to
// (x, -z, y), and sn columns 0:3 alike (S >= 3; the other columns stay); it is exact in any precision.  Before it, the
// detector's height scaling (oxford_detector_loader.py:188-192, train mode) multiplies pc z in place, a float32 array
// times a Python float: fl32(z * fl32(hs)).  A node has no height step here: its FPS candidates were gathered scaled.
// Runs on the raw row or node before any augmentation; without USIP_PAIR_ENU_TO_CAM it does nothing.
constexpr int PG_HEIGHT_SCALED = USIP_PAIR_TRAIN | USIP_PAIR_HEIGHT_SCALE;

__device__ __forceinline__ void pg_enu_to_cam(int flags, double hs, float& y, float& z, float* sn, int S) {
  if (!(flags & USIP_PAIR_ENU_TO_CAM)) return;
  if ((flags & PG_HEIGHT_SCALED) == PG_HEIGHT_SCALED) z = __fmul_rn(z, (float)hs);
  const float t = y;
  y = -z; z = t;
  if (S >= 3) {
    const float s1 = sn[1];
    sn[1] = -sn[2]; sn[2] = s1;
  }
}

// transform_pc_pytorch (augmentation.py:231-245) of one dst point or node: the fp32 R as column vectors, then the fp32
// scale and shift.  RT = the transform's R in fp32, P the pair's params block.  sn is only rotated (pg_colvec alone).
__device__ __forceinline__ void pg_dst_transform(const float* RT, const double* P, float& x, float& y, float& z) {
  pg_colvec(x, y, z, RT);
  const float sc = (float)P[43];                   // float32 tensor * Python float
  x = __fmul_rn(x, sc); y = __fmul_rn(y, sc); z = __fmul_rn(z, sc);
  x = __fadd_rn(x, (float)P[40]); y = __fadd_rn(y, (float)P[41]); z = __fadd_rn(z, (float)P[42]);
}

// The device-mode jitter laws of one augment call: N(0, sigma^2) clipped at +-clip for pc, every sn column and nodes.
struct PgJitterLaws {
  double pc_sigma, pc_clip, sn_sigma, sn_clip, node_sigma, node_clip;
};

// KITTI / Oxford detector pairs (usip_pair_augment) and, with per_pair_switch, the indoor detector pairs
// (usip_indoor_pair_augment, data/match3d_detector_loader.py / scenenn_detector_loader.py): the same arithmetic, the
// laws and the sn column passed in.  per_pair_switch: pair b is augmented only when params[b, 45] != 0.
__global__ void __launch_bounds__(PG_AUG_THREADS)
pair_augment_kernel(const float* __restrict__ scans, int C, const int64_t* __restrict__ offsets,
                    const int32_t* __restrict__ scan_of_cloud, const int32_t* __restrict__ rows,
                    const float* __restrict__ nodes, const double* __restrict__ params,
                    const double* __restrict__ jit_pc, const double* __restrict__ jit_sn,
                    const double* __restrict__ jit_node, uint64_t seed, uint64_t step, int flags, int S, int sn_col,
                    PgJitterLaws law, int per_pair_switch, int N, int M, float* __restrict__ src_pc,
                    float* __restrict__ src_sn, float* __restrict__ src_node, float* __restrict__ dst_pc,
                    float* __restrict__ dst_sn, float* __restrict__ dst_node, float* __restrict__ R_out,
                    float* __restrict__ scale_out, float* __restrict__ shift_out) {
  const int c = blockIdx.y, b = c >> 1, side = c & 1;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const double* P = params + (int64_t)b * PG_PARAM_STRIDE;
  const bool train = (flags & USIP_PAIR_TRAIN) && (!per_pair_switch || P[PG_AUGMENT_SLOT] != 0.0);
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
    pg_enu_to_cam(flags, P[44], y, z, sn, S);      // Oxford only: height scale, then the camera frame
    if (train) {                                   // KittiLoader.augment, :182-212
      double j[4];
      pg_jitter_xyz(jit_pc, (int64_t)c * N + i, seed, step, c, i, PURPOSE_JIT_PC, law.pc_sigma, law.pc_clip, j);
      pg_augment_point(flags, P, P[27], j, S, x, y, z, sn);
      pg_jitter_sn(jit_sn, (int64_t)c * N + i, seed, step, c, i, S, law.sn_sigma, law.sn_clip, sn);
    }
    float* opc = side ? dst_pc : src_pc;
    float* osn = side ? dst_sn : src_sn;
    if (side == 1) {                               // transform_pc_pytorch, fp32, column vectors
      pg_dst_transform(RT, P, x, y, z);
      if (S >= 3) pg_colvec(sn[0], sn[1], sn[2], RT);
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
    pg_enu_to_cam(flags & ~USIP_PAIR_HEIGHT_SCALE, 1.0, y, z, nullptr, 0);
    if (train) {
      double j[4];
      pg_jitter_xyz(jit_node, (int64_t)c * M + i, seed, step, c, i, PURPOSE_JIT_NODE, law.node_sigma, law.node_clip,
                    j);
      pg_augment_node(flags, P, P[27], j, x, y, z);
    }
    float* ond = side ? dst_node : src_node;
    if (side == 1) pg_dst_transform(RT, P, x, y, z);
    ond[((int64_t)b * 3 + 0) * M + i] = x;
    ond[((int64_t)b * 3 + 1) * M + i] = y;
    ond[((int64_t)b * 3 + 2) * M + i] = z;
  }
}

// ModelNet sn (modelnet_shrec_loader.py:213-233): `sn_np = atomic_rotate(sn_np, .)` builds a new float64 array, so
// after any rotation sn stays float64 through jitter and scale (the node's chain without the shift); without one it is
// still the float32 slice, jittered in place and scaled in fp32.  sn is never shifted.
__device__ __forceinline__ void pg_modelnet_sn(int flags, const double* P, double sc, const double* j, float& x,
                                               float& y, float& z) {
  if (flags & PG_ANY_ROT) {
    pg_augment_node(flags & ~USIP_PAIR_TRANSLATION, P, sc, j, x, y, z);
  } else {
    x = (float)__dadd_rn((double)x, j[0]); y = (float)__dadd_rn((double)y, j[1]);
    z = (float)__dadd_rn((double)z, j[2]);
    const float scf = (float)sc;
    x = __fmul_rn(x, scf); y = __fmul_rn(y, scf); z = __fmul_rn(z, scf);
  }
}

// ModelNet pairs (ModelNet_Shrec_Loader.augment, modelnet_shrec_loader.py:182-243, then transform_pc_pytorch for dst).
// Both clouds of pair b subsample the same file independently but read ONE draw of every jitter array: row i of src and
// of dst gets the same numbers (jit_* are per pair, and Philox is keyed by b, not by the cloud).  pc and nodes follow
// the KITTI arithmetic with ModelNet's jitter laws; sn = columns 3:6, see pg_modelnet_sn.
__global__ void __launch_bounds__(PG_AUG_THREADS)
modelnet_pair_augment_kernel(const float* __restrict__ scans, int C, const int64_t* __restrict__ offsets,
                             const int32_t* __restrict__ scan_of_cloud, const int32_t* __restrict__ rows,
                             const float* __restrict__ nodes, const double* __restrict__ params,
                             const double* __restrict__ jit_pc, const double* __restrict__ jit_sn,
                             const double* __restrict__ jit_node, uint64_t seed, uint64_t step, int flags, int N, int M,
                             float* __restrict__ src_pc, float* __restrict__ src_sn, float* __restrict__ src_node,
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
    const float* p = scans + (offsets[scan_of_cloud[c]] + rows[(int64_t)c * N + i]) * C;
    float x = p[0], y = p[1], z = p[2], nx = p[3], ny = p[4], nz = p[5];
    if (train) {                                   // ModelNet_Shrec_Loader.augment, :182-243
      double j[4];
      pg_jitter_xyz(jit_pc, (int64_t)b * N + i, seed, step, b, i, PURPOSE_JIT_PC, 0.01, 0.05, j);
      pg_augment_point(flags, P, P[27], j, 0, x, y, z, nullptr);
      pg_jitter_xyz(jit_sn, (int64_t)b * N + i, seed, step, b, i, PURPOSE_JIT_SN, 0.01, 0.05, j);
      pg_modelnet_sn(flags, P, P[27], j, nx, ny, nz);
    }
    if (side == 1) {
      pg_dst_transform(RT, P, x, y, z);
      pg_colvec(nx, ny, nz, RT);
    }
    float* opc = (side ? dst_pc : src_pc) + (int64_t)b * 3 * N;
    float* osn = (side ? dst_sn : src_sn) + (int64_t)b * 3 * N;
    opc[i] = x; opc[N + i] = y; opc[2 * N + i] = z;
    osn[i] = nx; osn[N + i] = ny; osn[2 * N + i] = nz;
  }

  if (i < M) {
    const float* nd = nodes + (int64_t)c * 3 * M;
    float x = nd[i], y = nd[M + i], z = nd[2 * M + i];
    if (train) {
      double j[4];
      pg_jitter_xyz(jit_node, (int64_t)b * M + i, seed, step, b, i, PURPOSE_JIT_NODE, 0.04, 0.1, j);
      pg_augment_node(flags, P, P[27], j, x, y, z);
    }
    if (side == 1) pg_dst_transform(RT, P, x, y, z);
    float* ond = (side ? dst_node : src_node) + (int64_t)b * 3 * M;
    ond[i] = x; ond[M + i] = y; ond[2 * M + i] = z;
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
    pg_enu_to_cam(flags, 1.0, y, z, sn, S);        // Oxford only: the camera frame
    if (train) {
      double j[4];
      pg_jitter_xyz(jit_pc, (int64_t)c * N + i, seed, step, c, i, PURPOSE_JIT_PC, 0.04, 0.12, j);
      pg_augment_point(flags, P, P[27], j, S, x, y, z, sn);
      pg_jitter_sn(jit_sn, (int64_t)c * N + i, seed, step, c, i, S, 0.01, 0.05, sn);
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
    pg_enu_to_cam(flags, 1.0, y, z, nullptr, 0);
    if (train) {
      double j[4];
      pg_jitter_xyz(jit_node, (int64_t)c * M + i, seed, step, c, i, PURPOSE_JIT_NODE, 0.04, 0.12, j);
      pg_augment_node(flags, P, P[27], j, x, y, z);
    }
    float* ond = side ? pos_node : anc_node;
    ond[((int64_t)b * 3 + 0) * M + i] = x;
    ond[((int64_t)b * 3 + 1) * M + i] = y;
    ond[((int64_t)b * 3 + 2) * M + i] = z;
  }
}

// Test-set clouds (KittiTestLoader / OxfordTestLoader.__getitem__, then save_keypoints.py:275's noise): no
// augmentation, no dst.  The rows and nodes as they are, moved to the camera frame under USIP_PAIR_ENU_TO_CAM (after
// FPS, as the Oxford loader does); then `anc_pc + torch.randn(size) * sigma`, a float32 tensor times a Python float.
__global__ void __launch_bounds__(PG_AUG_THREADS)
test_cloud_gather_kernel(const float* __restrict__ scans, int C, const int64_t* __restrict__ offsets,
                         const int32_t* __restrict__ scan_of_cloud, const int32_t* __restrict__ rows,
                         const float* __restrict__ nodes, const float* __restrict__ noise, float sigma, uint64_t seed,
                         uint64_t step, int flags, int S, int N, int M, float* __restrict__ pc, float* __restrict__ sn_out,
                         float* __restrict__ node_out) {
  const int c = blockIdx.y, i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < N) {
    const float* p = scans + (offsets[scan_of_cloud[c]] + rows[(int64_t)c * N + i]) * C;
    float x = p[0], y = p[1], z = p[2];
    float sn[PG_MAX_S];
#pragma unroll
    for (int k = 0; k < PG_MAX_S; ++k) sn[k] = k < S ? p[3 + k] : 0.f;
    pg_enu_to_cam(flags, 1.0, y, z, sn, S);
    float* o = pc + (int64_t)c * 3 * N;
    if (sigma != 0.f) {
      float n[3];
      if (noise) {
#pragma unroll
        for (int k = 0; k < 3; ++k) n[k] = noise[((int64_t)c * 3 + k) * N + i];
      } else {
        const uint4 u = pg_random(seed, step, c, i, PURPOSE_NOISE, 0);
        double z0, z1, z2, z3;
        pg_normal2(u.x, u.y, z0, z1); pg_normal2(u.z, u.w, z2, z3);
        n[0] = (float)z0; n[1] = (float)z1; n[2] = (float)z2;
      }
      x = __fadd_rn(x, __fmul_rn(n[0], sigma));
      y = __fadd_rn(y, __fmul_rn(n[1], sigma));
      z = __fadd_rn(z, __fmul_rn(n[2], sigma));
    }
    o[i] = x; o[N + i] = y; o[2 * N + i] = z;
#pragma unroll
    for (int k = 0; k < PG_MAX_S; ++k)
      if (k < S) sn_out[((int64_t)c * S + k) * N + i] = sn[k];
  }
  if (i < M) {
    const float* nd = nodes + (int64_t)c * 3 * M;
    float x = nd[i], y = nd[M + i], z = nd[2 * M + i];
    pg_enu_to_cam(flags, 1.0, y, z, nullptr, 0);
    float* o = node_out + (int64_t)c * 3 * M;
    o[i] = x; o[M + i] = y; o[2 * M + i] = z;
  }
}

// ------------------------------------------------------------------------ SceneNN descriptor pairs (ICP'd anchor)
// data/scenenn_descriptor_loader.py's __getitem__ aligns the anchor to the positive with the pair's 4x4 ICP matrix T:
// anc_pc = hom2cart(T @ [x y z 1]^T), float64 from here on, and anc_sn[:, 0:3] the same map, written back into the
// float32 sn view.  np.dot goes through BLAS, whose summation order is unspecified; this is the order fixed here (the
// order of a dgemm micro-kernel): per output row r, the fused multiply-add chain over k = 0, 1, 2, 3 started by a plain
// product, the last term T[r, 3] * 1 (an FMA by 1 is one rounded add).  Then x/w, y/w, z/w with w the fourth row's
// chain, divided literally (w is exactly 1 only when T's last row is [0 0 0 1]).
__device__ __forceinline__ void pg_icp(const double* T, double x, double y, double z, double& X, double& Y, double& Z) {
  double h[4];
#pragma unroll
  for (int r = 0; r < 4; ++r)
    h[r] = __dadd_rn(__fma_rn(z, T[4 * r + 2], __fma_rn(y, T[4 * r + 1], __dmul_rn(x, T[4 * r]))), T[4 * r + 3]);
  X = __ddiv_rn(h[0], h[3]); Y = __ddiv_rn(h[1], h[3]); Z = __ddiv_rn(h[2], h[3]);
}

// FPS input of the SceneNN descriptor: pts[c, j, :] = float64 xyz of rows[c, cand[c, j]], ICP'd on the anchor side
// (c even, T = icp[c / 2]), the exact double of the fp32 row on the positive side.
__global__ void pair_gather_icp_f64_kernel(const float* __restrict__ scans, int C, const int64_t* __restrict__ offsets,
                                           const int32_t* __restrict__ scan_of_cloud, const int32_t* __restrict__ rows,
                                           const int32_t* __restrict__ cand, const double* __restrict__ icp,
                                           double* __restrict__ pts, int N, int n_cand) {
  const int c = blockIdx.y, j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n_cand) return;
  const int r = rows[(int64_t)c * N + cand[(int64_t)c * n_cand + j]];
  const float* p = scans + (offsets[scan_of_cloud[c]] + r) * C;
  double X = p[0], Y = p[1], Z = p[2];
  if ((c & 1) == 0) pg_icp(icp + (int64_t)(c >> 1) * 16, p[0], p[1], p[2], X, Y, Z);
  double* o = pts + ((int64_t)c * n_cand + j) * 3;
  o[0] = X; o[1] = Y; o[2] = Z;
}

// SceneNNDescriptorLoader.augment / augment_rot_only of one float64 point (the ICP'd anchor's pc, every node): the
// rotations (kind >= 1), then with the full augmentation (kind 2) the scale and, under USIP_PAIR_TRANSLATION, the
// shift.  The loader draws its jitter but never adds it, so there is no jitter term (not even a zero: x + 0.0 would
// turn -0.0 into +0.0).
__device__ __forceinline__ void pg_scenenn_f64(int flags, int kind, const double* P, double& X, double& Y, double& Z) {
  if (kind < 1) return;
#pragma unroll
  for (int r = 0; r < 3; ++r)
    if (flags & (USIP_PAIR_ROT_HORIZONTAL << r)) pg_rowvec(X, Y, Z, P + 9 * r);
  if (kind < 2) return;
  X = __dmul_rn(X, P[27]); Y = __dmul_rn(Y, P[27]); Z = __dmul_rn(Z, P[27]);
  if (flags & USIP_PAIR_TRANSLATION) { X = __dadd_rn(X, P[28]); Y = __dadd_rn(Y, P[29]); Z = __dadd_rn(Z, P[30]); }
}

// sn columns 0:3 under the rotations (kind >= 1): a float32 view, rounded after every rotation; never scaled or shifted
__device__ __forceinline__ void pg_scenenn_sn(int flags, int kind, const double* P, float* sn) {
  if (kind < 1) return;
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    if (!(flags & (USIP_PAIR_ROT_HORIZONTAL << r))) continue;
    double a = sn[0], bb = sn[1], cc = sn[2];
    pg_rowvec(a, bb, cc, P + 9 * r);
    sn[0] = (float)a; sn[1] = (float)bb; sn[2] = (float)cc;
  }
}

// SceneNN descriptor pairs (scenenn_descriptor_loader.py:__getitem__, then transform_pc_pytorch on the positive).  The
// pair's one set of rotations, scale and shift applies to both clouds; kind = params[b, 45] picks the augmentation:
// 2 augment (train split), 1 augment_rot_only (val), anything else none (test).  The anchor's pc is float64 from its
// ICP to the final cast; its sn[0:3] is ICP'd and rounded to fp32.  The positive's pc is the float32 slice until its
// first rotation (then float64); un-rotated, the full augmentation scales it in fp32 and shifts it as fl32(x + shift).
// Nodes are re-read as float64 FPS candidates (cand_pts[c, node_idx[c, i]]), so they stay float64 to the cast.
__global__ void __launch_bounds__(PG_AUG_THREADS)
scenenn_desc_pair_augment_kernel(const float* __restrict__ scans, int C, const int64_t* __restrict__ offsets,
                                 const int32_t* __restrict__ scan_of_cloud, const int32_t* __restrict__ rows,
                                 const double* __restrict__ icp, const double* __restrict__ cand_pts,
                                 const int32_t* __restrict__ node_idx, const double* __restrict__ params, int flags,
                                 int S, int N, int M, int n_cand, float* __restrict__ anc_pc, float* __restrict__ anc_sn,
                                 float* __restrict__ anc_node, float* __restrict__ pos_pc, float* __restrict__ pos_sn,
                                 float* __restrict__ pos_node, float* __restrict__ R_out, float* __restrict__ scale_out,
                                 float* __restrict__ shift_out) {
  const int c = blockIdx.y, b = c >> 1, side = c & 1;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const double* P = params + (int64_t)b * PG_PARAM_STRIDE;
  const double* T = icp + (int64_t)b * 16;
  const int kind = P[PG_AUGMENT_SLOT] == 2.0 ? 2 : (P[PG_AUGMENT_SLOT] == 1.0 ? 1 : 0);
  float RT[9];
#pragma unroll
  for (int k = 0; k < 9; ++k) RT[k] = (float)P[31 + k];

  if (side == 1 && blockIdx.x == 0) {
    if (threadIdx.x < 9) R_out[b * 9 + threadIdx.x] = RT[threadIdx.x];
    else if (threadIdx.x == 9) scale_out[b] = (float)P[43];
    else if (threadIdx.x < 13) shift_out[b * 3 + threadIdx.x - 10] = (float)P[40 + threadIdx.x - 10];
  }

  if (i < N) {
    const float* p = scans + (offsets[scan_of_cloud[c]] + rows[(int64_t)c * N + i]) * C;
    float x = p[0], y = p[1], z = p[2];
    float sn[PG_MAX_S];
#pragma unroll
    for (int k = 0; k < PG_MAX_S; ++k) sn[k] = k < S ? p[3 + k] : 0.f;
    if (side == 0) {                               // ICP'd, float64 to the cast
      double X, Y, Z;
      pg_icp(T, x, y, z, X, Y, Z);
      pg_scenenn_f64(flags, kind, P, X, Y, Z);
      x = (float)X; y = (float)Y; z = (float)Z;
      double a, bb, cc;
      pg_icp(T, sn[0], sn[1], sn[2], a, bb, cc);
      sn[0] = (float)a; sn[1] = (float)bb; sn[2] = (float)cc;
    } else if (kind >= 1 && (flags & PG_ANY_ROT)) {  // float64 after the first rotation
      double X = x, Y = y, Z = z;
      pg_scenenn_f64(flags, kind, P, X, Y, Z);
      x = (float)X; y = (float)Y; z = (float)Z;
    } else if (kind == 2) {                        // the float32 slice: fp32 scale, then fl32(x + shift)
      const float scf = (float)P[27];
      x = __fmul_rn(x, scf); y = __fmul_rn(y, scf); z = __fmul_rn(z, scf);
      if (flags & USIP_PAIR_TRANSLATION) {
        x = (float)__dadd_rn((double)x, P[28]); y = (float)__dadd_rn((double)y, P[29]);
        z = (float)__dadd_rn((double)z, P[30]);
      }
    }
    pg_scenenn_sn(flags, kind, P, sn);
    float* opc = side ? pos_pc : anc_pc;
    float* osn = side ? pos_sn : anc_sn;
    if (side == 1) {                               // transform_pc_pytorch, fp32, column vectors
      pg_dst_transform(RT, P, x, y, z);
      pg_colvec(sn[0], sn[1], sn[2], RT);
    }
    opc[((int64_t)b * 3 + 0) * N + i] = x;
    opc[((int64_t)b * 3 + 1) * N + i] = y;
    opc[((int64_t)b * 3 + 2) * N + i] = z;
#pragma unroll
    for (int k = 0; k < PG_MAX_S; ++k)
      if (k < S) osn[((int64_t)b * S + k) * N + i] = sn[k];
  }

  if (i < M) {
    const double* q = cand_pts + ((int64_t)c * n_cand + node_idx[(int64_t)c * M + i]) * 3;
    double X = q[0], Y = q[1], Z = q[2];
    pg_scenenn_f64(flags, kind, P, X, Y, Z);
    float x = (float)X, y = (float)Y, z = (float)Z;
    if (side == 1) pg_dst_transform(RT, P, x, y, z);
    float* ond = side ? pos_node : anc_node;
    ond[((int64_t)b * 3 + 0) * M + i] = x;
    ond[((int64_t)b * 3 + 1) * M + i] = y;
    ond[((int64_t)b * 3 + 2) * M + i] = z;
  }
}

// t[b, k, :] *= f in fp32 (torch's `t[:, k, :] *= f` with f a Python float: fl32(v * fl32(f)))
__global__ void scale_channel_kernel(float* __restrict__ t, int C, int L, int k, float f) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= L) return;
  float* row = t + ((int64_t)blockIdx.y * C + k) * L;
  row[i] = __fmul_rn(row[i], f);
}

}  // namespace usip

using namespace usip;

static int pg_subset_smem(int n) { return n * (int)sizeof(uint32_t); }

// the longest scan pair_subset_kernel keeps in shared memory (one 31-bit key per row); also the largest N
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
  USIP_REQUIRE(max_rows <= USIP_SUBSAMPLE_MAX_ROWS, "cloud_subsample: a scan may have at most 16777216 rows");
  USIP_REQUIRE(N <= usip_pair_max_scan_rows(), "cloud_subsample: N too large for shared memory");
  const bool one_cta = max_rows <= usip_pair_max_scan_rows();
  cudaError_t e = cudaFuncSetAttribute(pair_subset_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       pg_subset_smem(one_cta ? max(max_rows, N) : N));
  if (e != cudaSuccess) { set_last_error("cloud_subsample: smem attribute"); return (int)e; }
  cudaStream_t s = (cudaStream_t)stream;
  int rc;
  if (one_cta) {
    pair_subset_kernel<<<2 * n_pairs, PG_THREADS, pg_subset_smem(max_rows), s>>>(
        scans, C, offsets, scan_of_cloud, 0, use_radius, radius, N, n_cand, seed, step, out_rows, out_cand, out_start,
        out_valid);
    rc = check_launch("pair_subset_kernel(rows)");
  } else {
    pair_subset_cluster_kernel<<<2 * n_pairs * PG_CLUSTER, PG_THREADS, 0, s>>>(
        scans, C, offsets, scan_of_cloud, use_radius, radius, N, seed, step, out_rows, out_valid);
    rc = check_launch("pair_subset_cluster_kernel(rows)");
  }
  if (rc) return rc;
  pair_subset_kernel<<<2 * n_pairs, PG_THREADS, pg_subset_smem(N), s>>>(
      scans, C, offsets, scan_of_cloud, 1, 0, 0.0, N, n_cand, seed, step, out_rows, out_cand, out_start, out_valid);
  return check_launch("pair_subset_kernel(candidates)");
}

static int pg_gather(const float* scans, int C, const int64_t* offsets, const int32_t* scan_of_cloud,
                     const int32_t* rows, const int32_t* cand, const float* z_scale, float* out_pts, int n_pairs, int N,
                     int n_cand, void* stream) {
  USIP_REQUIRE(scans && offsets && scan_of_cloud && rows && cand && out_pts, "cloud_gather_candidates: null pointer");
  USIP_REQUIRE(C >= 3 && n_pairs > 0 && N > 0 && n_cand > 0 && n_cand <= N, "cloud_gather_candidates: bad sizes");
  USIP_REQUIRE(n_pairs <= PG_MAX_PAIRS, "cloud_gather_candidates: at most 32767 pairs");
  dim3 grid(cdiv(n_cand, 256), 2 * n_pairs);
  pair_gather_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(scans, C, offsets, scan_of_cloud, rows, cand, z_scale,
                                                              out_pts, N, n_cand);
  return check_launch("pair_gather_kernel");
}

extern "C" int usip_cloud_gather_candidates(const float* scans, int C, const int64_t* offsets,
                                            const int32_t* scan_of_cloud, const int32_t* rows, const int32_t* cand,
                                            float* out_pts, int n_pairs, int N, int n_cand, void* stream) {
  return pg_gather(scans, C, offsets, scan_of_cloud, rows, cand, nullptr, out_pts, n_pairs, N, n_cand, stream);
}

extern "C" int usip_cloud_gather_candidates_zscaled(const float* scans, int C, const int64_t* offsets,
                                                    const int32_t* scan_of_cloud, const int32_t* rows,
                                                    const int32_t* cand, const float* z_scale, float* out_pts,
                                                    int n_pairs, int N, int n_cand, void* stream) {
  USIP_REQUIRE(z_scale, "cloud_gather_candidates_zscaled: null z_scale");
  return pg_gather(scans, C, offsets, scan_of_cloud, rows, cand, z_scale, out_pts, n_pairs, N, n_cand, stream);
}

extern "C" int usip_cloud_gather_candidates_icp_f64(const float* scans, int C, const int64_t* offsets,
                                                    const int32_t* scan_of_cloud, const int32_t* rows,
                                                    const int32_t* cand, const double* icp, double* out_pts,
                                                    int n_pairs, int N, int n_cand, void* stream) {
  USIP_REQUIRE(scans && offsets && scan_of_cloud && rows && cand && icp && out_pts,
               "cloud_gather_candidates_icp_f64: null pointer");
  USIP_REQUIRE(C >= 3 && n_pairs > 0 && N > 0 && n_cand > 0 && n_cand <= N,
               "cloud_gather_candidates_icp_f64: bad sizes");
  USIP_REQUIRE(n_pairs <= PG_MAX_PAIRS, "cloud_gather_candidates_icp_f64: at most 32767 pairs");
  dim3 grid(cdiv(n_cand, 256), 2 * n_pairs);
  pair_gather_icp_f64_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(scans, C, offsets, scan_of_cloud, rows, cand, icp,
                                                                      out_pts, N, n_cand);
  return check_launch("pair_gather_icp_f64_kernel");
}

extern "C" int usip_scenenn_desc_pair_augment(const float* scans, int C, const int64_t* offsets,
                                              const int32_t* scan_of_cloud, const int32_t* rows, const double* icp,
                                              const double* cand_pts, const int32_t* node_idx, const double* params,
                                              int flags, int S, int n_pairs, int N, int M, int n_cand, float* anc_pc,
                                              float* anc_sn, float* anc_node, float* pos_pc, float* pos_sn,
                                              float* pos_node, float* R, float* scale, float* shift, void* stream) {
  USIP_REQUIRE(icp, "scenenn_desc_pair_augment: null icp");
  USIP_REQUIRE(scans && offsets && scan_of_cloud && rows && cand_pts && node_idx && params,
               "scenenn_desc_pair_augment: null input");
  USIP_REQUIRE(anc_pc && anc_sn && anc_node && pos_pc && pos_sn && pos_node && R && scale && shift,
               "scenenn_desc_pair_augment: null output");
  USIP_REQUIRE(S >= 3 && S <= PG_MAX_S && 3 + S <= C,
               "scenenn_desc_pair_augment: sn is columns 3:3+S (3 <= S <= 8, 3+S <= C)");
  USIP_REQUIRE(!(flags & (USIP_PAIR_ENU_TO_CAM | USIP_PAIR_HEIGHT_SCALE)),
               "scenenn_desc_pair_augment: the Oxford frame flags do not apply to indoor fragments");
  USIP_REQUIRE(n_pairs > 0 && N > 0 && M > 0 && n_cand > 0 && M <= n_cand, "scenenn_desc_pair_augment: bad sizes");
  USIP_REQUIRE(n_pairs <= PG_MAX_PAIRS, "scenenn_desc_pair_augment: at most 32767 pairs");
  dim3 grid(cdiv(max(N, M), PG_AUG_THREADS), 2 * n_pairs);
  scenenn_desc_pair_augment_kernel<<<grid, PG_AUG_THREADS, 0, (cudaStream_t)stream>>>(
      scans, C, offsets, scan_of_cloud, rows, icp, cand_pts, node_idx, params, flags, S, N, M, n_cand, anc_pc, anc_sn,
      anc_node, pos_pc, pos_sn, pos_node, R, scale, shift);
  return check_launch("scenenn_desc_pair_augment_kernel");
}

extern "C" int usip_scale_channel_f32(float* t, int B, int C, int L, int k, float factor, void* stream) {
  USIP_REQUIRE(t, "scale_channel: null pointer");
  USIP_REQUIRE(B > 0 && C > 0 && L > 0 && k >= 0 && k < C && B <= 65535, "scale_channel: bad sizes");
  dim3 grid(cdiv(L, 256), B);
  scale_channel_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(t, C, L, k, factor);
  return check_launch("scale_channel_kernel");
}

extern "C" int usip_test_cloud_gather(const float* scans, int C, const int64_t* offsets, const int32_t* scan_of_cloud,
                                      const int32_t* rows, const float* nodes, const float* noise, float noise_sigma,
                                      uint64_t seed, uint64_t step, int flags, int S, int n_clouds, int N, int M,
                                      float* pc, float* sn, float* node, void* stream) {
  USIP_REQUIRE(scans && offsets && scan_of_cloud && rows && nodes, "test_cloud_gather: null input");
  USIP_REQUIRE(pc && sn && node, "test_cloud_gather: null output");
  USIP_REQUIRE(S >= 1 && S <= PG_MAX_S && 3 + S <= C, "test_cloud_gather: bad surface-normal length");
  USIP_REQUIRE((flags & ~USIP_PAIR_ENU_TO_CAM) == 0, "test_cloud_gather: only USIP_PAIR_ENU_TO_CAM applies");
  USIP_REQUIRE(!(flags & USIP_PAIR_ENU_TO_CAM) || S >= 3, "test_cloud_gather: the camera frame needs S >= 3");
  USIP_REQUIRE(n_clouds > 0 && n_clouds <= 65535 && N > 0 && M > 0, "test_cloud_gather: bad sizes");
  dim3 grid(cdiv(max(N, M), PG_AUG_THREADS), n_clouds);
  test_cloud_gather_kernel<<<grid, PG_AUG_THREADS, 0, (cudaStream_t)stream>>>(
      scans, C, offsets, scan_of_cloud, rows, nodes, noise, noise_sigma, seed, step, flags, S, N, M, pc, sn, node);
  return check_launch("test_cloud_gather_kernel");
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
  USIP_REQUIRE(!(flags & USIP_PAIR_HEIGHT_SCALE), "desc_pair_augment: no height scaling in the descriptor's clouds");
  USIP_REQUIRE(!(flags & USIP_PAIR_ENU_TO_CAM) || S >= 3, "desc_pair_augment: the camera frame needs S >= 3");
  USIP_REQUIRE(n_pairs > 0 && N > 0 && M > 0, "desc_pair_augment: bad sizes");
  USIP_REQUIRE(n_pairs <= PG_MAX_PAIRS, "desc_pair_augment: at most 32767 pairs");
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
  USIP_REQUIRE(!(flags & USIP_PAIR_ENU_TO_CAM) || S >= 3, "pair_augment: the camera frame needs S >= 3");
  USIP_REQUIRE(!(flags & USIP_PAIR_HEIGHT_SCALE) || (flags & USIP_PAIR_ENU_TO_CAM),
               "pair_augment: height scaling is part of the ENU frame step");
  USIP_REQUIRE(n_pairs > 0 && N > 0 && M > 0, "pair_augment: bad sizes");
  USIP_REQUIRE(n_pairs <= PG_MAX_PAIRS, "pair_augment: at most 32767 pairs");
  const int sn_col = S == 1 ? C - 1 : 3;           // kitti_detector_loader.py:135-139
  const PgJitterLaws kitti = {0.04, 0.12, 0.01, 0.05, 0.04, 0.12};   // kitti_detector_loader.py:164-172
  dim3 grid(cdiv(max(N, M), PG_AUG_THREADS), 2 * n_pairs);
  pair_augment_kernel<<<grid, PG_AUG_THREADS, 0, (cudaStream_t)stream>>>(
      scans, C, offsets, scan_of_cloud, rows, nodes, params, jit_pc, jit_sn, jit_node, seed, step, flags, S, sn_col,
      kitti, 0, N, M, src_pc, src_sn, src_node, dst_pc, dst_sn, dst_node, R, scale, shift);
  return check_launch("pair_augment_kernel");
}

extern "C" int usip_indoor_pair_augment(const float* scans, int C, const int64_t* offsets,
                                        const int32_t* scan_of_cloud, const int32_t* rows, const float* nodes,
                                        const double* params, const double* jit_pc, const double* jit_sn,
                                        const double* jit_node, uint64_t seed, uint64_t step, int flags, int S,
                                        int n_pairs, int N, int M, float* src_pc, float* src_sn, float* src_node,
                                        float* dst_pc, float* dst_sn, float* dst_node, float* R, float* scale,
                                        float* shift, void* stream) {
  USIP_REQUIRE(scans && offsets && scan_of_cloud && rows && nodes && params, "indoor_pair_augment: null input");
  USIP_REQUIRE(src_pc && src_sn && src_node && dst_pc && dst_sn && dst_node && R && scale && shift,
               "indoor_pair_augment: null output");
  USIP_REQUIRE(S >= 1 && S <= PG_MAX_S && 3 + S <= C, "indoor_pair_augment: sn is columns 3:3+S (1 <= S <= 8, 3+S <= C)");
  USIP_REQUIRE(!(flags & (USIP_PAIR_ENU_TO_CAM | USIP_PAIR_HEIGHT_SCALE)),
               "indoor_pair_augment: the Oxford frame flags do not apply to indoor fragments");
  USIP_REQUIRE(n_pairs > 0 && N > 0 && M > 0, "indoor_pair_augment: bad sizes");
  USIP_REQUIRE(n_pairs <= PG_MAX_PAIRS, "indoor_pair_augment: at most 32767 pairs");
  const PgJitterLaws indoor = {0.01, 0.02, 0.01, 0.02, 0.01, 0.02};  // match3d_detector_loader.py:125-132
  dim3 grid(cdiv(max(N, M), PG_AUG_THREADS), 2 * n_pairs);
  pair_augment_kernel<<<grid, PG_AUG_THREADS, 0, (cudaStream_t)stream>>>(
      scans, C, offsets, scan_of_cloud, rows, nodes, params, jit_pc, jit_sn, jit_node, seed, step, flags, S, 3, indoor,
      1, N, M, src_pc, src_sn, src_node, dst_pc, dst_sn, dst_node, R, scale, shift);
  return check_launch("pair_augment_kernel(indoor)");
}

extern "C" int usip_modelnet_pair_augment(const float* scans, int C, const int64_t* offsets,
                                          const int32_t* scan_of_cloud, const int32_t* rows, const float* nodes,
                                          const double* params, const double* jit_pc, const double* jit_sn,
                                          const double* jit_node, uint64_t seed, uint64_t step, int flags, int S,
                                          int n_pairs, int N, int M, float* src_pc, float* src_sn, float* src_node,
                                          float* dst_pc, float* dst_sn, float* dst_node, float* R, float* scale,
                                          float* shift, void* stream) {
  USIP_REQUIRE(scans && offsets && scan_of_cloud && rows && nodes && params, "modelnet_pair_augment: null input");
  USIP_REQUIRE(src_pc && src_sn && src_node && dst_pc && dst_sn && dst_node && R && scale && shift,
               "modelnet_pair_augment: null output");
  USIP_REQUIRE(S == 3 && C >= 6, "modelnet_pair_augment: sn is columns 3:6 (S == 3, C >= 6)");
  USIP_REQUIRE(n_pairs > 0 && N > 0 && M > 0, "modelnet_pair_augment: bad sizes");
  USIP_REQUIRE(n_pairs <= PG_MAX_PAIRS, "modelnet_pair_augment: at most 32767 pairs");
  dim3 grid(cdiv(max(N, M), PG_AUG_THREADS), 2 * n_pairs);
  modelnet_pair_augment_kernel<<<grid, PG_AUG_THREADS, 0, (cudaStream_t)stream>>>(
      scans, C, offsets, scan_of_cloud, rows, nodes, params, jit_pc, jit_sn, jit_node, seed, step, flags, N, M, src_pc,
      src_sn, src_node, dst_pc, dst_sn, dst_node, R, scale, shift);
  return check_launch("modelnet_pair_augment_kernel");
}
