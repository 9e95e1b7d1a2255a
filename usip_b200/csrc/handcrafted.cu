// handcrafted.cu -- the handcrafted keypoint baselines of evaluation/save_keypoints.py:44-63, 289-331: ISS (PCL
// ISSKeypoint3D, no border estimation), Harris-3D (PCL HarrisKeypoint3D, HARRIS response, no refinement) and the
// random selection, with ensure_keypoint_number's padding for a whole keypoint-count sweep.
//
// Every radius pass reads one cell grid per cloud (usip_hc_grid_build): nngrid.cu's multi-CTA bin/scatter with the
// cloud as its own query set, followed by hc_stable_kernel, which puts the entries of every cell in ascending row order.
// Neighbour rule of every pass: j in N_r(i) <=> d2 = (dx*dx + dy*dy) + dz*dz in fp32 without FMA and d2 <= fl(r*r);
// i is its own neighbour; a non-finite row is nobody's neighbour and never a keypoint.
//
// One warp per query walks the cells that cover [p - r, p + r] as one flattened candidate list (ng_query_kernel's form):
// no neighbour list is materialised and a neighbourhood has no size cap.  Each lane sums the candidates k = lane mod 32
// of that list and the lanes are combined by a fixed butterfly, so a sum's order depends on the cell contents only:
// repeated runs are bitwise equal, and two rows with equal coordinates get bitwise-equal scores.
#include "nngrid.cuh"

namespace usip {

constexpr int HC_THREADS = 256;                    // radius passes: 8 queries (warps) per CTA
constexpr int HC_SEL_THREADS = 1024;               // selection: one CTA per cloud

// ---------------------------------------------------------------------------------------------- the grid
// scratch: ng_build_layout (nngrid.cuh) | the stable copy of `sorted`, float4 [B][N]
struct HcGrid {
  NgBuild ng;
  float4* stable;
};

static size_t hc_grid_bytes(int B, int N) { return ng_build_bytes(B, N) + (size_t)B * N * sizeof(float4) + 16; }

static HcGrid hc_grid_layout(void* scratch, int B, int N) {
  HcGrid g;
  g.ng = ng_build_layout(scratch, B, N);
  const uintptr_t end = reinterpret_cast<uintptr_t>(g.ng.cellid + (size_t)B * N);
  g.stable = reinterpret_cast<float4*>((end + 15) & ~(uintptr_t)15);
  return g;
}

// Slot of sorted entry p inside its cell = the number of entries of that cell with a smaller row.
__global__ void __launch_bounds__(256)
hc_stable_kernel(const float4* __restrict__ sorted, const int32_t* __restrict__ cell_start,
                 const int32_t* __restrict__ cellid, const NgGrid* __restrict__ grids, int N, float4* __restrict__ out) {
  const int b = blockIdx.y, p = blockIdx.x * blockDim.x + threadIdx.x;
  const NgGrid g = ng_load_grid(grids + b);
  const int32_t* cs = cell_start + (size_t)b * (NG_MAXC + 1);
  if (p >= __ldg(cs + g.nx * g.ny * g.nz)) return;
  const float4* s = sorted + (size_t)b * N;
  const int* rows = reinterpret_cast<const int*>(s) + 3;             // .w of entry q at rows[4 * q]
  const float4 e = s[p];
  const int n = __float_as_int(e.w);
  const int c = __ldg(cellid + (size_t)b * N + n);
  const int c0 = __ldg(cs + c), c1 = __ldg(cs + c + 1);
  int rank = 0;
  for (int q = c0; q < c1; ++q) rank += __ldg(rows + 4 * (size_t)q) < n;
  out[(size_t)b * N + c0 + rank] = e;
}

// ---------------------------------------------------------------------------------------------- the radius walk
// Calls f(entry) on this lane for its share of the rows j in N_r(a).  The cells of [a - rr, a + rr] per axis, with rr
// a thousandth wider than r: fp32 rounding can let d2 <= r*r hold for an |dx| a few ulps above r, and the cell index is
// monotone in the coordinate, so every neighbour lies in those cells.
template <class F>
__device__ __forceinline__ void hc_walk(float ax, float ay, float az, float r, float r2, const NgGrid& g,
                                        const int32_t* __restrict__ cs, const float4* __restrict__ pts, int lane, F&& f) {
  const float rr = r * 1.001f;
  const int x0 = ng_cell1(ax - rr, g.ox, g.inv_h, g.nx), x1 = ng_cell1(ax + rr, g.ox, g.inv_h, g.nx);
  const int y0 = ng_cell1(ay - rr, g.oy, g.inv_h, g.ny), y1 = ng_cell1(ay + rr, g.oy, g.inv_h, g.ny);
  const int z0 = ng_cell1(az - rr, g.oz, g.inv_h, g.nz), z1 = ng_cell1(az + rr, g.oz, g.inv_h, g.nz);
  const int ny_r = y1 - y0 + 1, nrows = (z1 - z0 + 1) * ny_r;    // one (z, y) row of cells = one contiguous range
  for (int j0 = 0; j0 < nrows; j0 += 32) {
    const int j = j0 + lane;
    int s = 0, len = 0;
    if (j < nrows) {
      const int z = z0 + j / ny_r, y = y0 + j % ny_r, base = (z * g.ny + y) * g.nx;
      s = __ldg(cs + base + x0);
      len = __ldg(cs + base + x1 + 1) - s;
    }
    int incl = len;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const int v = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += v; }
    const int total = __shfl_sync(0xffffffffu, incl, 31);
    const int excl = incl - len;
    for (int k0 = 0; k0 < total; k0 += 32) {
      const int k = k0 + lane;
      int lo = 0;
#pragma unroll
      for (int step = 16; step > 0; step >>= 1) {
        const int v = __shfl_sync(0xffffffffu, incl, lo + step - 1);
        if (k >= v) lo += step;
      }
      const int sj = __shfl_sync(0xffffffffu, s, lo), ej = __shfl_sync(0xffffffffu, excl, lo);
      if (k < total) {
        const float4 p = __ldg(pts + sj + (k - ej));
        if (sqdist_rn(ax, ay, az, p.x, p.y, p.z) <= r2) f(p);
      }
    }
  }
}

__device__ __forceinline__ int warp_sum_i(int v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// ---------------------------------------------------------------------------------------------- 3x3 eigen-analysis
// Cyclic Jacobi on a symmetric 3x3 in fp64: rotation (p, q) zeroes a[p][q] (Numerical Recipes' jacobi, written as
// c, s rotations).  Accurate to a few ulps of the largest eigenvalue; deterministic.
__device__ __forceinline__ void hc_jacobi_rot(double a[3][3], double v[3][3], int p, int q) {
  const double apq = a[p][q];
  if (apq == 0.0) return;
  const double theta = (a[q][q] - a[p][p]) / (2.0 * apq);
  double t = 1.0 / (fabs(theta) + sqrt(theta * theta + 1.0));
  if (theta < 0.0) t = -t;
  const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
  a[p][p] -= t * apq;
  a[q][q] += t * apq;
  a[p][q] = a[q][p] = 0.0;
  const int r = 3 - p - q;
  const double arp = a[r][p], arq = a[r][q];
  a[r][p] = a[p][r] = c * arp - s * arq;
  a[r][q] = a[q][r] = s * arp + c * arq;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const double vp = v[k][p], vq = v[k][q];
    v[k][p] = c * vp - s * vq;
    v[k][q] = s * vp + c * vq;
  }
}

// m = (xx, xy, xz, yy, yz, zz) -> w descending, v[:, k] the unit eigenvector of w[k].
__device__ void hc_eig3(const double m[6], double w[3], double v[3][3]) {
  double a[3][3] = {{m[0], m[1], m[2]}, {m[1], m[3], m[4]}, {m[2], m[4], m[5]}};
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) v[i][j] = i == j ? 1.0 : 0.0;
  for (int sweep = 0; sweep < 32; ++sweep) {
    const double off = fabs(a[0][1]) + fabs(a[0][2]) + fabs(a[1][2]);
    const double dia = fabs(a[0][0]) + fabs(a[1][1]) + fabs(a[2][2]);
    if (!(off > 1e-30 * dia)) break;                              // also stops on a NaN matrix
    hc_jacobi_rot(a, v, 0, 1);
    hc_jacobi_rot(a, v, 0, 2);
    hc_jacobi_rot(a, v, 1, 2);
  }
  int o[3] = {0, 1, 2};
  double d[3] = {a[0][0], a[1][1], a[2][2]};
  auto cs = [&](int i, int j) { if (d[o[i]] < d[o[j]]) { const int t = o[i]; o[i] = o[j]; o[j] = t; } };
  cs(0, 1); cs(1, 2); cs(0, 1);
  double vv[3][3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    w[k] = d[o[k]];
#pragma unroll
    for (int i = 0; i < 3; ++i) vv[i][k] = v[i][o[k]];
  }
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int k = 0; k < 3; ++k) v[i][k] = vv[i][k];
}

__device__ __forceinline__ void hc_reduce6(double c[6]) {
#pragma unroll
  for (int k = 0; k < 6; ++k) c[k] = warp_sum_d(c[k]);
}

// ---------------------------------------------------------------------------------------------- ISS saliency
__global__ void __launch_bounds__(HC_THREADS)
hc_iss_kernel(const float* __restrict__ pc, int N, int total, const float4* __restrict__ pts,
              const int32_t* __restrict__ cell_start, const NgGrid* __restrict__ grids, float r, float r2, double g21,
              double g32, int min_neighbors, double* __restrict__ saliency, int32_t* __restrict__ count,
              double* __restrict__ eig) {
  const int q = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (q >= total) return;
  const int b = q / N, i = q - b * N;
  const float* p = pc + (size_t)b * 3 * N;
  const float ax = __ldg(p + i), ay = __ldg(p + N + i), az = __ldg(p + 2 * N + i);
  const bool fin = ng_finite3(ax, ay, az);
  int cnt = 0;
  double c[6] = {0, 0, 0, 0, 0, 0};
  if (fin) {
    const NgGrid g = ng_load_grid(grids + b);
    hc_walk(ax, ay, az, r, r2, g, cell_start + (size_t)b * (NG_MAXC + 1), pts + (size_t)b * N, lane, [&](float4 e) {
      const double dx = (double)e.x - (double)ax, dy = (double)e.y - (double)ay, dz = (double)e.z - (double)az;
      ++cnt;
      c[0] += dx * dx; c[1] += dx * dy; c[2] += dx * dz; c[3] += dy * dy; c[4] += dy * dz; c[5] += dz * dz;
    });
    cnt = warp_sum_i(cnt);
    hc_reduce6(c);
  }
  if (lane != 0) return;
  double w[3] = {0, 0, 0}, s = 0.0;
  if (fin) {
    double v[3][3];
    hc_eig3(c, w, v);
    if (cnt >= min_neighbors && w[1] / w[0] < g21 && w[2] / w[1] < g32 && w[2] >= 0.0) s = w[2];
  }
  saliency[q] = s;
  if (count) count[q] = cnt;
  if (eig) { eig[3 * (size_t)q] = w[0]; eig[3 * (size_t)q + 1] = w[1]; eig[3 * (size_t)q + 2] = w[2]; }
}

// ---------------------------------------------------------------------------------------------- Harris-3D
// Normal: eigenvector of the smallest eigenvalue of the mean-centred covariance of N_r(i), NaN below 3 neighbours.
__global__ void __launch_bounds__(HC_THREADS)
hc_normal_kernel(const float* __restrict__ pc, int N, int total, const float4* __restrict__ pts,
                 const int32_t* __restrict__ cell_start, const NgGrid* __restrict__ grids, float r, float r2,
                 double* __restrict__ normals, int32_t* __restrict__ count) {
  const int q = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (q >= total) return;
  const int b = q / N, i = q - b * N;
  const float* p = pc + (size_t)b * 3 * N;
  const float ax = __ldg(p + i), ay = __ldg(p + N + i), az = __ldg(p + 2 * N + i);
  const bool fin = ng_finite3(ax, ay, az);
  int cnt = 0;
  double s1[3] = {0, 0, 0}, c[6] = {0, 0, 0, 0, 0, 0};
  if (fin) {
    const NgGrid g = ng_load_grid(grids + b);
    hc_walk(ax, ay, az, r, r2, g, cell_start + (size_t)b * (NG_MAXC + 1), pts + (size_t)b * N, lane, [&](float4 e) {
      const double dx = (double)e.x - (double)ax, dy = (double)e.y - (double)ay, dz = (double)e.z - (double)az;
      ++cnt;
      s1[0] += dx; s1[1] += dy; s1[2] += dz;
      c[0] += dx * dx; c[1] += dx * dy; c[2] += dx * dz; c[3] += dy * dy; c[4] += dy * dz; c[5] += dz * dz;
    });
    cnt = warp_sum_i(cnt);
#pragma unroll
    for (int k = 0; k < 3; ++k) s1[k] = warp_sum_d(s1[k]);
    hc_reduce6(c);
  }
  if (lane != 0) return;
  double n[3] = {NAN, NAN, NAN};
  if (fin && cnt >= 3) {
    const double inv = 1.0 / (double)cnt;
    const double m[3] = {s1[0] * inv, s1[1] * inv, s1[2] * inv};
    const double cov[6] = {c[0] * inv - m[0] * m[0], c[1] * inv - m[0] * m[1], c[2] * inv - m[0] * m[2],
                           c[3] * inv - m[1] * m[1], c[4] * inv - m[1] * m[2], c[5] * inv - m[2] * m[2]};
    double w[3], v[3][3];
    hc_eig3(cov, w, v);
    n[0] = v[0][2]; n[1] = v[1][2]; n[2] = v[2][2];
  }
  normals[3 * (size_t)q] = n[0]; normals[3 * (size_t)q + 1] = n[1]; normals[3 * (size_t)q + 2] = n[2];
  if (count) count[q] = cnt;
}

// Response: A = mean of n_j n_j^T over j in N_r(i) with a finite normal (NaN without one); R = 0.04 + det(A) -
// 0.04 trace(A)^2 when trace(A) != 0, else 0 (PCL's responseHarris).  NaN for a non-finite row.
__global__ void __launch_bounds__(HC_THREADS)
hc_harris_kernel(const float* __restrict__ pc, int N, int total, const float4* __restrict__ pts,
                 const int32_t* __restrict__ cell_start, const NgGrid* __restrict__ grids, float r, float r2,
                 const double* __restrict__ normals, double* __restrict__ response) {
  const int q = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (q >= total) return;
  const int b = q / N, i = q - b * N;
  const float* p = pc + (size_t)b * 3 * N;
  const float ax = __ldg(p + i), ay = __ldg(p + N + i), az = __ldg(p + 2 * N + i);
  const bool fin = ng_finite3(ax, ay, az);
  int cnt = 0;
  double c[6] = {0, 0, 0, 0, 0, 0};
  if (fin) {
    const NgGrid g = ng_load_grid(grids + b);
    const double* nb = normals + (size_t)b * N * 3;
    hc_walk(ax, ay, az, r, r2, g, cell_start + (size_t)b * (NG_MAXC + 1), pts + (size_t)b * N, lane, [&](float4 e) {
      const int j = __float_as_int(e.w);
      const double nx = __ldg(nb + 3 * j), ny = __ldg(nb + 3 * j + 1), nz = __ldg(nb + 3 * j + 2);
      if (nx == nx) {                                              // normals are all-NaN or finite
        ++cnt;
        c[0] += nx * nx; c[1] += nx * ny; c[2] += nx * nz; c[3] += ny * ny; c[4] += ny * nz; c[5] += nz * nz;
      }
    });
    cnt = warp_sum_i(cnt);
    hc_reduce6(c);
  }
  if (lane != 0) return;
  double R = NAN;
  if (fin && cnt > 0) {
    const double inv = 1.0 / (double)cnt;
    const double a0 = c[0] * inv, a1 = c[1] * inv, a2 = c[2] * inv, a3 = c[3] * inv, a4 = c[4] * inv, a5 = c[5] * inv;
    const double tr = a0 + a3 + a5;
    const double det = a0 * a3 * a5 + 2.0 * a1 * a2 * a4 - a2 * a2 * a3 - a1 * a1 * a5 - a4 * a4 * a0;
    R = tr != 0.0 ? 0.04 + det - 0.04 * tr * tr : 0.0;
  }
  response[q] = R;
}

// ---------------------------------------------------------------------------------------------- non-maximum test
// flag_i = p_i finite, s_i eligible (s_i > thr when strict, s_i >= thr otherwise; NaN never), |N_r(i)| >= min_count and
// no j in N_r(i) with s_j > s_i (a NaN s_j never suppresses).
__global__ void __launch_bounds__(HC_THREADS)
hc_nonmax_kernel(const float* __restrict__ pc, int N, int total, const float4* __restrict__ pts,
                 const int32_t* __restrict__ cell_start, const NgGrid* __restrict__ grids, float r, float r2,
                 const double* __restrict__ score, double thr, int strict, int min_count, int32_t* __restrict__ flag,
                 int32_t* __restrict__ count) {
  const int q = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (q >= total) return;
  const int b = q / N, i = q - b * N;
  const float* p = pc + (size_t)b * 3 * N;
  const float ax = __ldg(p + i), ay = __ldg(p + N + i), az = __ldg(p + 2 * N + i);
  const bool fin = ng_finite3(ax, ay, az);
  const double si = __ldg(score + q);
  const bool elig = fin && (strict ? si > thr : si >= thr);
  int cnt = 0;
  bool beaten = false;
  if (fin && (elig || count)) {
    const NgGrid g = ng_load_grid(grids + b);
    const double* sb = score + (size_t)b * N;
    hc_walk(ax, ay, az, r, r2, g, cell_start + (size_t)b * (NG_MAXC + 1), pts + (size_t)b * N, lane, [&](float4 e) {
      ++cnt;
      beaten |= __ldg(sb + __float_as_int(e.w)) > si;
    });
    cnt = warp_sum_i(cnt);
    beaten = __any_sync(0xffffffffu, beaten);
  }
  if (lane != 0) return;
  flag[q] = (elig && cnt >= min_count && !beaten) ? 1 : 0;
  if (count) count[q] = cnt;
}

// ---------------------------------------------------------------------------------------------- selection
// The `need` smallest u = (Philox word << 32 | row) over the rows with flag != 0 (every row without flags), ascending,
// to out[0..need).  u is unique per row, so an eight-pass radix select finds the need-th smallest exactly; the chosen
// ones are gathered in shared memory and bitonic-sorted.
__device__ __forceinline__ uint64_t hc_key(uint64_t seed, uint64_t step, int c, int i, int purpose) {
  return ((uint64_t)pg_random(seed, step, c, i, purpose, 0).x << 32) | (uint32_t)i;
}

__device__ void hc_select_band(const int32_t* __restrict__ fl, int N, int need, uint64_t seed, uint64_t step, int c,
                               int purpose, uint64_t* list, uint32_t* hist, uint32_t* s_ctl, int32_t* __restrict__ out) {
  if (need <= 0) return;
  const int tid = threadIdx.x, lane = tid & 31;
  uint64_t prefix = 0, pmask = 0;
  uint32_t rem = (uint32_t)need;
  for (int shift = 56; shift >= 0; shift -= 8) {
    for (int k = tid; k < 256; k += blockDim.x) hist[k] = 0;
    __syncthreads();
    for (int i = tid; i < N; i += blockDim.x) {
      if (fl && !fl[i]) continue;
      const uint64_t u = hc_key(seed, step, c, i, purpose);
      if ((u & pmask) == prefix) atomicAdd(&hist[(u >> shift) & 255u], 1u);
    }
    __syncthreads();
    if (tid < 32) {                                                // bin holding the rem-th smallest, rank inside it
      uint32_t loc[8], s = 0;
#pragma unroll
      for (int j = 0; j < 8; ++j) { loc[j] = hist[lane * 8 + j]; s += loc[j]; }
      uint32_t inc = s;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) { const uint32_t t = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += t; }
      uint32_t run = inc - s;
      if (run < rem && rem <= inc) {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          if (run < rem && rem <= run + loc[j]) { s_ctl[0] = (uint32_t)(lane * 8 + j); s_ctl[1] = rem - run; }
          run += loc[j];
        }
      }
    }
    __syncthreads();
    prefix |= (uint64_t)s_ctl[0] << shift;
    pmask |= 0xffull << shift;
    rem = s_ctl[1];
    __syncthreads();
  }
  if (tid == 0) s_ctl[0] = 0;
  __syncthreads();
  for (int i = tid; i < N; i += blockDim.x) {
    if (fl && !fl[i]) continue;
    const uint64_t u = hc_key(seed, step, c, i, purpose);
    if (u <= prefix) list[atomicAdd(&s_ctl[0], 1u)] = u;
  }
  int P = 1;
  while (P < need) P <<= 1;
  __syncthreads();
  for (int i = need + tid; i < P; i += blockDim.x) list[i] = ~0ull;
  __syncthreads();
  for (int k = 2; k <= P; k <<= 1)
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = tid; i < P; i += blockDim.x) {
        const int ixj = i ^ j;
        if (ixj > i) {
          const uint64_t x = list[i], y = list[ixj];
          if ((x > y) == ((i & k) == 0)) { list[i] = y; list[ixj] = x; }
        }
      }
      __syncthreads();
    }
  for (int i = tid; i < need; i += blockDim.x) out[i] = (int32_t)(uint32_t)list[i];
  __syncthreads();
}

__global__ void __launch_bounds__(HC_SEL_THREADS)
hc_select_kernel(const int32_t* __restrict__ flag, int N, int L, uint64_t seed, uint64_t step, int32_t* __restrict__ order,
                 int32_t* __restrict__ count) {
  __shared__ uint64_t list[USIP_HC_MAX_SELECT];
  __shared__ uint32_t hist[256];
  __shared__ uint32_t s_ctl[2];
  __shared__ int s_n;
  const int b = blockIdx.x, tid = threadIdx.x;
  const int32_t* fl = flag ? flag + (size_t)b * N : nullptr;
  if (tid == 0) s_n = 0;
  __syncthreads();
  if (fl) {
    int my = 0;
    for (int i = tid; i < N; i += blockDim.x) my += fl[i] != 0;
    my = warp_sum_i(my);
    if ((tid & 31) == 0 && my) atomicAdd(&s_n, my);
  }
  __syncthreads();
  const int nflag = s_n;
  if (tid == 0) count[b] = nflag;
  const int need1 = min(nflag, L);
  int32_t* o = order + (size_t)b * L;
  hc_select_band(fl, N, need1, seed, step, b, PURPOSE_HC_KEYPOINT, list, hist, s_ctl, o);
  hc_select_band(nullptr, N, L - need1, seed, step, b, PURPOSE_HC_PAD, list, hist, s_ctl, o + need1);
}

// ---------------------------------------------------------------------------------------------- host helpers
static bool hc_radius_ok(float r) { return r > 0.f && r <= 3.0e38f; }
static bool hc_shape_ok(int B, int N) {
  return B > 0 && N > 0 && N <= USIP_HC_MAX_POINTS && B <= 65535 && (int64_t)B * N <= USIP_HC_MAX_TOTAL;
}

}  // namespace usip

using namespace usip;

extern "C" size_t usip_hc_grid_scratch_bytes(int B, int N) {
  if (!hc_shape_ok(B, N)) return 0;
  return hc_grid_bytes(B, N);
}

#define HC_CHECK_GRID(name)                                                                                       \
  USIP_REQUIRE(pc && grid && hc_shape_ok(B, N), name ": bad args (B, N in range?)");                             \
  USIP_REQUIRE(grid_bytes >= hc_grid_bytes(B, N), name ": grid scratch too small");                               \
  USIP_REQUIRE((reinterpret_cast<uintptr_t>(grid) & 15) == 0, name ": grid scratch must be 16-byte aligned")

extern "C" int usip_hc_grid_build(const float* pc, void* grid, size_t grid_bytes, int B, int N, void* stream) {
  HC_CHECK_GRID("hc_grid_build");
  cudaStream_t st = (cudaStream_t)stream;
  const HcGrid g = hc_grid_layout(grid, B, N);
  const int e = ng_build_multi(pc, N, pc, N, B, g.ng, st);
  if (e != 0) return e;
  hc_stable_kernel<<<dim3(cdiv(N, 256), B), 256, 0, st>>>(g.ng.sorted, g.ng.cell_start, g.ng.cellid, g.ng.grids, N,
                                                          g.stable);
  return check_launch("hc_stable_kernel");
}

extern "C" int usip_iss_saliency_f64(const float* pc, const void* grid, size_t grid_bytes, int B, int N,
                                     float salient_radius, double gamma_21, double gamma_32, int min_neighbors,
                                     double* saliency, int32_t* count, double* eig, void* stream) {
  HC_CHECK_GRID("iss_saliency");
  USIP_REQUIRE(saliency, "iss_saliency: saliency is NULL");
  USIP_REQUIRE(hc_radius_ok(salient_radius), "iss_saliency: salient_radius must be finite and > 0");
  USIP_REQUIRE(gamma_21 > 0.0 && gamma_21 <= 1.0 && gamma_32 > 0.0 && gamma_32 <= 1.0,
               "iss_saliency: gamma_21 and gamma_32 must lie in (0, 1]");
  USIP_REQUIRE(min_neighbors >= 1, "iss_saliency: min_neighbors must be >= 1");
  const HcGrid g = hc_grid_layout(const_cast<void*>(grid), B, N);
  const int total = B * N;
  hc_iss_kernel<<<cdiv(total, HC_THREADS / 32), HC_THREADS, 0, (cudaStream_t)stream>>>(
      pc, N, total, g.stable, g.ng.cell_start, g.ng.grids, salient_radius, salient_radius * salient_radius,
      gamma_21, gamma_32, min_neighbors, saliency, count, eig);
  return check_launch("hc_iss_kernel");
}

extern "C" int usip_harris3d_response_f64(const float* pc, const void* grid, size_t grid_bytes, int B, int N,
                                          float radius, double* normals, double* response, int32_t* count,
                                          void* stream) {
  HC_CHECK_GRID("harris3d_response");
  USIP_REQUIRE(normals && response, "harris3d_response: normals or response is NULL");
  USIP_REQUIRE(hc_radius_ok(radius), "harris3d_response: radius must be finite and > 0");
  const HcGrid g = hc_grid_layout(const_cast<void*>(grid), B, N);
  const int total = B * N;
  cudaStream_t st = (cudaStream_t)stream;
  const float r2 = radius * radius;
  hc_normal_kernel<<<cdiv(total, HC_THREADS / 32), HC_THREADS, 0, st>>>(pc, N, total, g.stable, g.ng.cell_start,
                                                                        g.ng.grids, radius, r2, normals, count);
  hc_harris_kernel<<<cdiv(total, HC_THREADS / 32), HC_THREADS, 0, st>>>(pc, N, total, g.stable, g.ng.cell_start,
                                                                        g.ng.grids, radius, r2, normals, response);
  return check_launch("hc_harris_kernel");
}

extern "C" int usip_hc_nonmax(const float* pc, const void* grid, size_t grid_bytes, int B, int N, const double* score,
                              float radius, double threshold, int strict, int min_neighbors, int32_t* flag,
                              int32_t* count, void* stream) {
  HC_CHECK_GRID("hc_nonmax");
  USIP_REQUIRE(score && flag, "hc_nonmax: score or flag is NULL");
  USIP_REQUIRE(hc_radius_ok(radius), "hc_nonmax: radius must be finite and > 0");
  USIP_REQUIRE(threshold == threshold, "hc_nonmax: threshold is NaN");
  USIP_REQUIRE(min_neighbors >= 1, "hc_nonmax: min_neighbors must be >= 1");
  const HcGrid g = hc_grid_layout(const_cast<void*>(grid), B, N);
  const int total = B * N;
  hc_nonmax_kernel<<<cdiv(total, HC_THREADS / 32), HC_THREADS, 0, (cudaStream_t)stream>>>(
      pc, N, total, g.stable, g.ng.cell_start, g.ng.grids, radius, radius * radius, score, threshold,
      strict ? 1 : 0, min_neighbors, flag, count);
  return check_launch("hc_nonmax_kernel");
}

extern "C" int usip_hc_select(const int32_t* flag, int B, int N, int L, uint64_t seed, uint64_t step, int32_t* order,
                              int32_t* count, void* stream) {
  USIP_REQUIRE(order && count && hc_shape_ok(B, N), "hc_select: bad args (B, N in range?)");
  USIP_REQUIRE(L >= 1 && L <= N, "hc_select: need 1 <= L <= N");
  USIP_REQUIRE(L <= USIP_HC_MAX_SELECT, "hc_select: L above USIP_HC_MAX_SELECT");
  hc_select_kernel<<<B, HC_SEL_THREADS, 0, (cudaStream_t)stream>>>(flag, N, L, seed, step, order, count);
  return check_launch("hc_select_kernel");
}
