// nngrid.cu -- exact nearest neighbour through a per-cloud cell grid (cubic cells, counting-sorted entries).
//
// Two users on the detector path, both replacing brute-force scans that sat at their fp32-issue bound:
//   * usip_pairwise_min_grid_f32: the "keypoint on point cloud" searches of the loss (models/keypoint_detector.py:187-197 ->
//     losses.py:125-143: min_j ||kp_i - pc_j||, 512 keypoints against 16384 points per cloud).  The cloud is binned by many
//     CTAs (ng_bin_kernel / ng_scatter_kernel), one warp per keypoint walks the cell shells (ng_query_kernel).
//   * usip_som_assign_grid_f32: nearest node of every point (util/som.py:17-54, k = 1).  The <= 1024 nodes are sorted by one
//     CTA per cloud (ng_build_kernel) and staged in shared memory, one thread per point searches (ng_assign_kernel).
// A search scans the cells of ring r = 0, 1, ... around the query and stops when the best distance is provably smaller than
// anything outside the scanned cube.
//
// Same arithmetic and tie rule as the brute-force kernels (csrc/loss.cu, csrc/group.cu): d2 = (dx*dx + dy*dy) + dz*dz without
// FMA, smaller distance first, then smaller index; non-finite entries are never selected (their d2 is NaN or inf, which
// `d < best` rejects in the reference formulation as well); a query with no selectable entry yields (inf, 0) / node 0.
#include "nngrid.cuh"

namespace usip {

constexpr int NG_BT = 1024;            // build threads
constexpr int NG_MAXRING = 6;          // shells scanned before a query falls back to the whole (sorted) cloud

// One CTA per cloud.  sorted[b][0..cnt) = (x, y, z, bits(n)) grouped by cell (x fastest), cell_start[b][0..ncell].
__global__ void __launch_bounds__(NG_BT)
ng_build_kernel(const float* __restrict__ pts, int N, float4* __restrict__ sorted, int32_t* __restrict__ cell_start,
                NgGrid* __restrict__ grids, int max_cells) {
  extern __shared__ int ng_sm[];                                 // start[NG_MAXC + 1] | fill[NG_MAXC]
  int* start = ng_sm;
  int* fill = ng_sm + NG_MAXC + 1;
  __shared__ float red[6][NG_BT / 32];
  __shared__ NgGrid sg;
  __shared__ int wsum[NG_BT / 32];
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const float* px = pts + (size_t)b * 3 * N;
  const float* py = px + N;
  const float* pz = py + N;
  // ---- bounding box of the finite points
  float lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
  for (int n = tid; n < N; n += NG_BT) {
    const float x = px[n], y = py[n], z = pz[n];
    if (ng_finite3(x, y, z)) {
      lo[0] = fminf(lo[0], x); lo[1] = fminf(lo[1], y); lo[2] = fminf(lo[2], z);
      hi[0] = fmaxf(hi[0], x); hi[1] = fmaxf(hi[1], y); hi[2] = fmaxf(hi[2], z);
    }
  }
#pragma unroll
  for (int a = 0; a < 3; ++a) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      lo[a] = fminf(lo[a], __shfl_xor_sync(0xffffffffu, lo[a], o));
      hi[a] = fmaxf(hi[a], __shfl_xor_sync(0xffffffffu, hi[a], o));
    }
    if (lane == 0) { red[a][warp] = lo[a]; red[3 + a][warp] = hi[a]; }
  }
  for (int c = tid; c < NG_MAXC; c += NG_BT) fill[c] = 0;
  __syncthreads();
  if (tid == 0) {
    float l[3], h3[3];
    for (int a = 0; a < 3; ++a) {
      l[a] = INFINITY; h3[a] = -INFINITY;
      for (int w = 0; w < NG_BT / 32; ++w) { l[a] = fminf(l[a], red[a][w]); h3[a] = fmaxf(h3[a], red[3 + a][w]); }
    }
    NgGrid g;
    if (!(l[0] <= h3[0])) {                                      // no finite point at all
      g.ox = g.oy = g.oz = 0.f; g.h = 1.f; g.inv_h = 1.f; g.nx = g.ny = g.nz = 1;
    } else {
      const float ex = h3[0] - l[0], ey = h3[1] - l[1], ez = h3[2] - l[2];
      const float me = fmaxf(ex, fmaxf(ey, ez));
      float h = me > 0.f ? me / (float)NG_AXIS : 1.f;
      if (!(h >= 1e-30f) || !(h <= 3.0e38f)) h = fmaxf(fminf(h, 3.0e38f), 1e-30f);
      int nx, ny, nz;
      for (int it = 0; it < 64; ++it) {
        nx = min(NG_AXIS, (int)(ex / h) + 1); ny = min(NG_AXIS, (int)(ey / h) + 1); nz = min(NG_AXIS, (int)(ez / h) + 1);
        if ((long long)nx * ny * nz <= max_cells) break;
        h *= 1.25f;
      }
      if ((long long)nx * ny * nz > max_cells) { nx = ny = nz = 1; h = fmaxf(me, 1e-30f) * 2.f; }
      g.ox = l[0]; g.oy = l[1]; g.oz = l[2]; g.h = h; g.inv_h = 1.f / h; g.nx = nx; g.ny = ny; g.nz = nz;
    }
    sg = g;
    grids[b] = g;
  }
  __syncthreads();
  const NgGrid g = sg;
  const int ncell = g.nx * g.ny * g.nz;
  // ---- histogram
  for (int n = tid; n < N; n += NG_BT) {
    const float x = px[n], y = py[n], z = pz[n];
    if (ng_finite3(x, y, z)) {
      const int c = (ng_cell1(z, g.oz, g.inv_h, g.nz) * g.ny + ng_cell1(y, g.oy, g.inv_h, g.ny)) * g.nx + ng_cell1(x, g.ox, g.inv_h, g.nx);
      atomicAdd(&fill[c], 1);
    }
  }
  __syncthreads();
  // ---- exclusive scan over the cells (8 per thread)
  constexpr int PER = NG_MAXC / NG_BT;
  int loc[PER], s = 0;
#pragma unroll
  for (int j = 0; j < PER; ++j) { const int c = tid * PER + j; loc[j] = c < ncell ? fill[c] : 0; s += loc[j]; }
  int inc = s;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const int v = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += v; }
  if (lane == 31) wsum[warp] = inc;
  __syncthreads();
  if (warp == 0) {
    int v = wsum[lane];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const int u = __shfl_up_sync(0xffffffffu, v, o); if (lane >= o) v += u; }
    wsum[lane] = v;
  }
  __syncthreads();
  int run = inc - s + (warp > 0 ? wsum[warp - 1] : 0);
  int32_t* cs = cell_start + (size_t)b * (NG_MAXC + 1);
#pragma unroll
  for (int j = 0; j < PER; ++j) {
    const int c = tid * PER + j;
    if (c < ncell) { start[c] = run; cs[c] = run; }
    run += loc[j];
  }
  if (tid == NG_BT - 1) { start[ncell] = run; cs[ncell] = run; }
  __syncthreads();
  for (int c = tid; c < ncell; c += NG_BT) fill[c] = 0;
  __syncthreads();
  // ---- scatter (order inside a cell is arbitrary; the query's (d2, index) rule does not depend on it)
  float4* out = sorted + (size_t)b * N;
  for (int n = tid; n < N; n += NG_BT) {
    const float x = px[n], y = py[n], z = pz[n];
    if (ng_finite3(x, y, z)) {
      const int c = (ng_cell1(z, g.oz, g.inv_h, g.nz) * g.ny + ng_cell1(y, g.oy, g.inv_h, g.ny)) * g.nx + ng_cell1(x, g.ox, g.inv_h, g.nx);
      const int pos = start[c] + atomicAdd(&fill[c], 1);
      out[pos] = make_float4(x, y, z, __int_as_float(n));
    }
  }
}

// ---- the same structure for a LARGE cloud, built by many CTAs (the one-CTA build above moves the whole cloud through one
// SM: 33 us for 16384 points).  The grid is derived from the bounding box of the QUERIES -- a few hundred values that every
// CTA reduces for itself -- and cloud points outside it are clamped into the border cells (the search never uses a grid
// border as a distance bound, so clamping keeps it exact).  bin: cell id per point + global histogram; scatter: prefix of the
// histogram (scanned by every CTA for itself) + fill[cell]++ gives the slot.  Both counter arrays are zeroed by one memset
// node ahead of the launches.
constexpr int NGB_THREADS = 256;
constexpr int NGB_PTS = 4;

__device__ __forceinline__ NgGrid ng_grid_from_box(const float* l, const float* h3, int max_cells) {
  NgGrid g;
  if (!(l[0] <= h3[0])) {                                        // no finite value at all
    g.ox = g.oy = g.oz = 0.f; g.h = 1.f; g.inv_h = 1.f; g.nx = g.ny = g.nz = 1;
    return g;
  }
  const float ex = h3[0] - l[0], ey = h3[1] - l[1], ez = h3[2] - l[2];
  const float me = fmaxf(ex, fmaxf(ey, ez));
  float h = me > 0.f ? me / (float)NG_AXIS : 1.f;
  if (!(h >= 1e-30f) || !(h <= 3.0e38f)) h = fmaxf(fminf(h, 3.0e38f), 1e-30f);
  int nx = 1, ny = 1, nz = 1;
  for (int it = 0; it < 64; ++it) {
    nx = min(NG_AXIS, (int)(ex / h) + 1); ny = min(NG_AXIS, (int)(ey / h) + 1); nz = min(NG_AXIS, (int)(ez / h) + 1);
    if ((long long)nx * ny * nz <= max_cells) break;
    h *= 1.25f;
  }
  if ((long long)nx * ny * nz > max_cells) { nx = ny = nz = 1; h = fmaxf(me, 1e-30f) * 2.f; }
  g.ox = l[0]; g.oy = l[1]; g.oz = l[2]; g.h = h; g.inv_h = 1.f / h; g.nx = nx; g.ny = ny; g.nz = nz;
  return g;
}

__global__ void __launch_bounds__(NGB_THREADS)
ng_bin_kernel(const float* __restrict__ qry, int Ma, const float* __restrict__ pts, int N, int32_t* __restrict__ cellid,
              int32_t* __restrict__ cnt, NgGrid* __restrict__ grids) {
  __shared__ float red[6][NGB_THREADS / 32];
  __shared__ NgGrid sg;
  const int b = blockIdx.y, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const float* qx = qry + (size_t)b * 3 * Ma;
  float lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
  for (int i = tid; i < Ma; i += NGB_THREADS) {
    const float x = __ldg(qx + i), y = __ldg(qx + Ma + i), z = __ldg(qx + 2 * Ma + i);
    if (ng_finite3(x, y, z)) {
      lo[0] = fminf(lo[0], x); lo[1] = fminf(lo[1], y); lo[2] = fminf(lo[2], z);
      hi[0] = fmaxf(hi[0], x); hi[1] = fmaxf(hi[1], y); hi[2] = fmaxf(hi[2], z);
    }
  }
  // the points of this CTA are fetched while the box is reduced
  const float* px = pts + (size_t)b * 3 * N;
  float x[NGB_PTS], y[NGB_PTS], z[NGB_PTS];
  const int n0 = blockIdx.x * (NGB_THREADS * NGB_PTS) + tid;
#pragma unroll
  for (int j = 0; j < NGB_PTS; ++j) {
    const int n = n0 + j * NGB_THREADS;
    const bool ok = n < N;
    x[j] = ok ? __ldg(px + n) : NAN; y[j] = ok ? __ldg(px + N + n) : NAN; z[j] = ok ? __ldg(px + 2 * N + n) : NAN;
  }
#pragma unroll
  for (int a = 0; a < 3; ++a) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      lo[a] = fminf(lo[a], __shfl_xor_sync(0xffffffffu, lo[a], o));
      hi[a] = fmaxf(hi[a], __shfl_xor_sync(0xffffffffu, hi[a], o));
    }
    if (lane == 0) { red[a][warp] = lo[a]; red[3 + a][warp] = hi[a]; }
  }
  __syncthreads();
  if (tid == 0) {
    float l[3], h3[3];
    for (int a = 0; a < 3; ++a) {
      l[a] = INFINITY; h3[a] = -INFINITY;
      for (int w = 0; w < NGB_THREADS / 32; ++w) { l[a] = fminf(l[a], red[a][w]); h3[a] = fmaxf(h3[a], red[3 + a][w]); }
    }
    sg = ng_grid_from_box(l, h3, NG_MAXC);
    if (blockIdx.x == 0) grids[b] = sg;
  }
  __syncthreads();
  const NgGrid g = sg;
  int32_t* cb = cnt + (size_t)b * (NG_MAXC + 1);
#pragma unroll
  for (int j = 0; j < NGB_PTS; ++j) {
    const int n = n0 + j * NGB_THREADS;
    if (n < N) {
      int c = -1;
      if (ng_finite3(x[j], y[j], z[j])) {
        c = (ng_cell1(z[j], g.oz, g.inv_h, g.nz) * g.ny + ng_cell1(y[j], g.oy, g.inv_h, g.ny)) * g.nx + ng_cell1(x[j], g.ox, g.inv_h, g.nx);
        atomicAdd(cb + c, 1);
      }
      cellid[(size_t)b * N + n] = c;
    }
  }
}

// Every CTA scans the cloud's histogram for itself in shared memory (32 KB of L2-resident counters, ~1 us, all CTAs at once)
// instead of waiting for a one-CTA-per-cloud scan launch (12 us under ncu) or for a last-CTA tail (which ran at the memory
// parallelism of a single CTA: 15-40 us).  CTA 0 of a cloud publishes cell_start[] for the query kernel.
constexpr int NGS_PTS = 8;            // points per scatter thread: 33 KB of shared memory per CTA -> half the CTAs, one wave
__global__ void __launch_bounds__(NGB_THREADS)
ng_scatter_kernel(const float* __restrict__ pts, int N, const int32_t* __restrict__ cellid, const int32_t* __restrict__ cnt,
                  int32_t* __restrict__ fill, const NgGrid* __restrict__ grids, int32_t* __restrict__ cell_start,
                  float4* __restrict__ sorted) {
  extern __shared__ int ngs_start[];                             // [NG_MAXC + NG_MAXC / 32] padded: index k -> k + (k >> 5)
  __shared__ int wsum[NGB_THREADS / 32];
  const int b = blockIdx.y, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const NgGrid g = ng_load_grid(grids + b);
  const int ncell = g.nx * g.ny * g.nz;
  const int32_t* cb = cnt + (size_t)b * (NG_MAXC + 1);
  // the points of this CTA are fetched while the histogram is scanned
  const float* px = pts + (size_t)b * 3 * N;
  const int n0 = blockIdx.x * (NGB_THREADS * NGS_PTS) + tid;
  float x[NGS_PTS], y[NGS_PTS], z[NGS_PTS]; int c[NGS_PTS];
#pragma unroll
  for (int j = 0; j < NGS_PTS; ++j) {
    const int n = n0 + j * NGB_THREADS;
    const bool ok = n < N;
    c[j] = ok ? __ldg(cellid + (size_t)b * N + n) : -1;
    x[j] = ok ? __ldg(px + n) : 0.f; y[j] = ok ? __ldg(px + N + n) : 0.f; z[j] = ok ? __ldg(px + 2 * N + n) : 0.f;
  }
  for (int k = tid; k < NG_MAXC; k += NGB_THREADS) ngs_start[k + (k >> 5)] = k < ncell ? __ldg(cb + k) : 0;   // coalesced
  __syncthreads();
  constexpr int PER = NG_MAXC / NGB_THREADS;                     // 32 consecutive cells per thread; the padding spreads the banks
  const int k0 = tid * PER;
  int s = 0;
#pragma unroll
  for (int j = 0; j < PER; ++j) s += ngs_start[k0 + j + ((k0 + j) >> 5)];
  int inc = s;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const int v = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += v; }
  if (lane == 31) wsum[warp] = inc;
  __syncthreads();
  int run = inc - s;
  for (int w2 = 0; w2 < warp; ++w2) run += wsum[w2];
  int32_t* cs = cell_start + (size_t)b * (NG_MAXC + 1);
  const bool publish = blockIdx.x == 0;
#pragma unroll
  for (int j = 0; j < PER; ++j) {
    const int k = k0 + j, idx = k + (k >> 5);
    const int v = ngs_start[idx];
    ngs_start[idx] = run;
    if (publish && k < ncell) cs[k] = run;
    run += v;
  }
  if (publish && tid == NGB_THREADS - 1) cs[ncell] = run;
  __syncthreads();
  int32_t* fl = fill + (size_t)b * (NG_MAXC + 1);
  float4* out = sorted + (size_t)b * N;
#pragma unroll
  for (int j = 0; j < NGS_PTS; ++j)
    if (c[j] >= 0) {
      const int pos = ngs_start[c[j] + (c[j] >> 5)] + atomicAdd(fl + c[j], 1);
      out[pos] = make_float4(x[j], y[j], z[j], __int_as_float(n0 + j * NGB_THREADS));
    }
}

// Shell search of ONE thread around (ax, ay, az): cells of ring r = 0, 1, ... until the best squared distance is smaller than
// the distance to everything outside the scanned cube (the warp-per-query kernel below has its own, flattened form).
// (best, bidx) = lexicographic minimum of (d2, original index).
__device__ __forceinline__ void ng_search(float ax, float ay, float az, const NgGrid g, const int32_t* cs, const float4* pts,
                                          int cnt, float& best, int& bidx) {
  auto scan = [&](int s, int e) {
    for (int t = s; t < e; ++t) {
      const float4 p = pts[t];
      const float d = sqdist_rn(ax, ay, az, p.x, p.y, p.z);
      const int n = __float_as_int(p.w);
      if (d < best || (d == best && n < bidx)) { best = d; bidx = n; }
    }
  };
  const int cx = ng_cell1(ax, g.ox, g.inv_h, g.nx), cy = ng_cell1(ay, g.oy, g.inv_h, g.ny), cz = ng_cell1(az, g.oz, g.inv_h, g.nz);
  bool done = false;
  for (int r = 0; r <= NG_MAXRING && !done; ++r) {
    const int z0 = max(cz - r, 0), z1 = min(cz + r, g.nz - 1), y0 = max(cy - r, 0), y1 = min(cy + r, g.ny - 1);
    const int x0 = max(cx - r, 0), x1 = min(cx + r, g.nx - 1);
    for (int z = z0; z <= z1; ++z) {
      for (int y = y0; y <= y1; ++y) {
        const int row = (z * g.ny + y) * g.nx;
        if (z == cz - r || z == cz + r || y == cy - r || y == cy + r) {          // a face row of the shell: whole x range
          scan(cs[row + x0], cs[row + x1 + 1]);
        } else {                                                                 // interior row: the two end cells
          if (cx - r >= 0) scan(cs[row + cx - r], cs[row + cx - r + 1]);
          if (cx + r < g.nx && r > 0) scan(cs[row + cx + r], cs[row + cx + r + 1]);
        }
      }
    }
    // everything outside the cube of half-width r is at least `lb` away (faces beyond the grid do not count)
    float lb = INFINITY;
    if (cx - r > 0) lb = fminf(lb, ax - (g.ox + (float)(cx - r) * g.h));
    if (cx + r < g.nx - 1) lb = fminf(lb, (g.ox + (float)(cx + r + 1) * g.h) - ax);
    if (cy - r > 0) lb = fminf(lb, ay - (g.oy + (float)(cy - r) * g.h));
    if (cy + r < g.ny - 1) lb = fminf(lb, (g.oy + (float)(cy + r + 1) * g.h) - ay);
    if (cz - r > 0) lb = fminf(lb, az - (g.oz + (float)(cz - r) * g.h));
    if (cz + r < g.nz - 1) lb = fminf(lb, (g.oz + (float)(cz + r + 1) * g.h) - az);
    if (lb == INFINITY) { done = true; break; }                   // the cube covers the grid: every point was seen
    lb = fmaxf(lb - 1e-3f * g.h, 0.f);                            // cell assignment rounds: keep a margin of h/1000
    if (best < lb * lb) done = true;
  }
  if (!done) scan(0, cnt);                                        // far query: the whole sorted set (duplicates are harmless)
}

// One warp per query.  The cell ranges of a shell are fetched by all lanes at once (lane = one range: a face row's whole x
// span, or one end cell of an interior row), then the candidates of up to 32 ranges are walked as ONE flattened list -- a
// warp prefix sum over the range lengths, a 5-step shuffle search for the owner of candidate k -- so a ring costs two
// dependent memory round trips (cell bounds, then points) however its points are spread over the cells.
__device__ __forceinline__ void ng_warp_ranges(int s, int len, int lane, const float4* __restrict__ pts, float ax, float ay,
                                               float az, float& best, int& bidx) {
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
      const float d = sqdist_rn(ax, ay, az, p.x, p.y, p.z);
      const int n = __float_as_int(p.w);
      if (d < best || (d == best && n < bidx)) { best = d; bidx = n; }
    }
  }
}

__global__ void __launch_bounds__(256)
ng_query_kernel(const float* __restrict__ a, int Ma, const float4* __restrict__ sorted, const int32_t* __restrict__ cell_start,
                const NgGrid* __restrict__ grids, int N, float* __restrict__ min_d, int32_t* __restrict__ arg, int total) {
  const int q = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (q >= total) return;
  const int b = q / Ma, i = q - b * Ma;
  const float* pa = a + (size_t)b * 3 * Ma;
  const float ax = __ldg(pa + i), ay = __ldg(pa + Ma + i), az = __ldg(pa + 2 * Ma + i);
  const NgGrid g = ng_load_grid(grids + b);
  const int32_t* cs = cell_start + (size_t)b * (NG_MAXC + 1);
  const float4* pts = sorted + (size_t)b * N;
  const int cnt = __ldg(cs + g.nx * g.ny * g.nz);
  float best = INFINITY; int bidx = 0x7fffffff;
  auto reduce = [&]() {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ob = __shfl_xor_sync(0xffffffffu, best, o); const int oi = __shfl_xor_sync(0xffffffffu, bidx, o);
      if (ob < best || (ob == best && oi < bidx)) { best = ob; bidx = oi; }
    }
  };
  if (ng_finite3(ax, ay, az) && cnt > 0) {
    const int cx = ng_cell1(ax, g.ox, g.inv_h, g.nx), cy = ng_cell1(ay, g.oy, g.inv_h, g.ny), cz = ng_cell1(az, g.oz, g.inv_h, g.nz);
    bool done = false;
    for (int r = 1; r <= NG_MAXRING && !done; ++r) {             // r = 1 scans the whole 3x3x3 cube, r > 1 the shell only
      const int z0 = max(cz - r, 0), z1 = min(cz + r, g.nz - 1), y0 = max(cy - r, 0), y1 = min(cy + r, g.ny - 1);
      const int x0 = max(cx - r, 0), x1 = min(cx + r, g.nx - 1);
      const int ny_r = y1 - y0 + 1, nslots = 2 * (z1 - z0 + 1) * ny_r;     // two range slots per (z, y) row
      for (int j0 = 0; j0 < nslots; j0 += 32) {
        const int j = j0 + lane;
        int s = 0, len = 0;
        if (j < nslots) {
          const int row = j >> 1, which = j & 1, z = z0 + row / ny_r, y = y0 + row % ny_r;
          const int base = (z * g.ny + y) * g.nx;
          const bool face = (r == 1) || z == cz - r || z == cz + r || y == cy - r || y == cy + r;
          int ca = -1, cb = -1;                                   // cells [ca, cb] of this row
          if (face) { if (which == 0) { ca = x0; cb = x1; } }
          else if (which == 0) { if (cx - r >= 0) ca = cb = cx - r; }
          else { if (cx + r < g.nx) ca = cb = cx + r; }
          if (ca >= 0) { s = __ldg(cs + base + ca); len = __ldg(cs + base + cb + 1) - s; }
        }
        ng_warp_ranges(s, len, lane, pts, ax, ay, az, best, bidx);
      }
      reduce();
      // everything outside the cube of half-width r is at least `lb` away (faces beyond the grid do not count)
      float lb = INFINITY;
      if (cx - r > 0) lb = fminf(lb, ax - (g.ox + (float)(cx - r) * g.h));
      if (cx + r < g.nx - 1) lb = fminf(lb, (g.ox + (float)(cx + r + 1) * g.h) - ax);
      if (cy - r > 0) lb = fminf(lb, ay - (g.oy + (float)(cy - r) * g.h));
      if (cy + r < g.ny - 1) lb = fminf(lb, (g.oy + (float)(cy + r + 1) * g.h) - ay);
      if (cz - r > 0) lb = fminf(lb, az - (g.oz + (float)(cz - r) * g.h));
      if (cz + r < g.nz - 1) lb = fminf(lb, (g.oz + (float)(cz + r + 1) * g.h) - az);
      if (lb == INFINITY) { done = true; break; }                 // the cube covers the grid: every point was seen
      lb = fmaxf(lb - 1e-3f * g.h, 0.f);                          // cell assignment rounds: keep a margin of h/1000
      if (best < lb * lb) done = true;
    }
    if (!done) {                                                  // far query: the whole sorted cloud (duplicates are harmless)
      for (int t = lane; t < cnt; t += 32) {
        const float4 p = __ldg(pts + t);
        const float d = sqdist_rn(ax, ay, az, p.x, p.y, p.z);
        const int n = __float_as_int(p.w);
        if (d < best || (d == best && n < bidx)) { best = d; bidx = n; }
      }
      reduce();
    }
  }
  if (lane == 0) {
    const bool none = !(best < INFINITY);
    const size_t o = (size_t)b * Ma + i;
    if (min_d) min_d[o] = none ? INFINITY : __fsqrt_rn(best);
    if (arg) arg[o] = none ? 0 : bidx;
  }
}

// Nearest node of every point (som.query_topk k = 1, util/som.py:17-54): the grid holds the M nodes of the cloud, staged in
// shared memory; one thread per point.  min_idx = smallest m among the nearest nodes, 0 when no node is selectable
// (exactly what the brute-force scan leaves behind); count[b, m] += 1.
constexpr int NGA_THREADS = 256;
constexpr int NGA_MAXM = 1024;         // nodes per cloud the shared-memory copy holds
constexpr int NGA_MAXC = 1024;         // cells of the node grid

__global__ void __launch_bounds__(NGA_THREADS)
ng_assign_kernel(const float* __restrict__ xyz, int N, int M, const float4* __restrict__ sorted,
                 const int32_t* __restrict__ cell_start, const NgGrid* __restrict__ grids, int32_t* __restrict__ min_idx,
                 int32_t* __restrict__ count) {
  __shared__ float4 snode[NGA_MAXM];
  __shared__ int32_t scs[NGA_MAXC + 1];
  const int b = blockIdx.y;
  const NgGrid g = ng_load_grid(grids + b);
  const int ncell = g.nx * g.ny * g.nz;
  const int32_t* cs = cell_start + (size_t)b * (NG_MAXC + 1);
  for (int c = threadIdx.x; c <= ncell; c += NGA_THREADS) scs[c] = cs[c];
  __syncthreads();
  const int cnt = scs[ncell];
  for (int t = threadIdx.x; t < cnt; t += NGA_THREADS) snode[t] = sorted[(size_t)b * M + t];
  __syncthreads();
  const int n = blockIdx.x * NGA_THREADS + threadIdx.x;
  if (n >= N) return;
  const float* px = xyz + (size_t)b * 3 * N;
  const float x = px[n], y = px[N + n], z = px[2 * N + n];
  float best = INFINITY; int bi = 0x7fffffff;
  if (ng_finite3(x, y, z) && cnt > 0) ng_search(x, y, z, g, scs, snode, cnt, best, bi);
  if (!(best < INFINITY)) bi = 0;
  min_idx[(size_t)b * N + n] = bi;
  if (count) atomicAdd(&count[(size_t)b * M + bi], 1);
}

// ---- the multi-CTA build as one call (usip_pairwise_min_grid_f32, handcrafted.cu)
size_t ng_build_bytes(int B, int N) {
  return (size_t)B * N * sizeof(float4) + 3 * (size_t)B * (NG_MAXC + 1) * sizeof(int32_t) + (size_t)B * sizeof(NgGrid) +
         (size_t)B * N * sizeof(int32_t) + 128;
}

NgBuild ng_build_layout(void* scratch, int B, int N) {
  NgBuild s;
  s.sorted = reinterpret_cast<float4*>(scratch);
  s.cell_start = reinterpret_cast<int32_t*>(s.sorted + (size_t)B * N);
  NgGrid* grids = reinterpret_cast<NgGrid*>(s.cell_start + (size_t)B * (NG_MAXC + 1));
  s.grids = reinterpret_cast<NgGrid*>((reinterpret_cast<uintptr_t>(grids) + 15) & ~(uintptr_t)15);
  s.cnt = reinterpret_cast<int32_t*>(s.grids + B);
  s.fill = s.cnt + (size_t)B * (NG_MAXC + 1);
  s.cellid = s.fill + (size_t)B * (NG_MAXC + 1);
  return s;
}

int ng_build_multi(const float* qry, int Ma, const float* pts, int N, int B, const NgBuild& s, cudaStream_t st) {
  cudaError_t e = cudaMemsetAsync(s.cnt, 0, 2 * (size_t)B * (NG_MAXC + 1) * sizeof(int32_t), st);
  if (e != cudaSuccess) { set_last_error("grid build: memset"); return (int)e; }
  static bool attr = false;
  const size_t smem = (size_t)(NG_MAXC + NG_MAXC / 32) * sizeof(int);
  if (!attr) {
    e = cudaFuncSetAttribute(ng_scatter_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) { set_last_error("grid build: smem attribute"); return (int)e; }
    attr = true;
  }
  const dim3 pgrid(cdiv(N, NGB_THREADS * NGB_PTS), B);
  ng_bin_kernel<<<pgrid, NGB_THREADS, 0, st>>>(qry, Ma, pts, N, s.cellid, s.cnt, s.grids);
  const dim3 sgrid(cdiv(N, NGB_THREADS * NGS_PTS), B);
  ng_scatter_kernel<<<sgrid, NGB_THREADS, smem, st>>>(pts, N, s.cellid, s.cnt, s.fill, s.grids, s.cell_start, s.sorted);
  return check_launch("grid build");
}

}  // namespace usip

using namespace usip;

// scratch layout: ng_build_layout (nngrid.cuh)
extern "C" size_t usip_pairwise_min_grid_scratch_bytes(int B, int Nb) {
  if (B <= 0 || Nb <= 0) return 0;
  return ng_build_bytes(B, Nb);
}

extern "C" int usip_pairwise_min_grid_f32(const float* a, const float* b, float* min_d, int32_t* arg, void* scratch,
                                          size_t scratch_bytes, int B, int Ma, int Nb, void* stream) {
  USIP_REQUIRE(a && b && scratch && B > 0 && Ma > 0 && Nb > 0, "pairwise_min_grid: bad args");
  USIP_REQUIRE(scratch_bytes >= usip_pairwise_min_grid_scratch_bytes(B, Nb), "pairwise_min_grid: scratch too small");
  USIP_REQUIRE((reinterpret_cast<uintptr_t>(scratch) & 15) == 0, "pairwise_min_grid: scratch must be 16-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  const NgBuild nb = ng_build_layout(scratch, B, Nb);
  const int e = ng_build_multi(a, Ma, b, Nb, B, nb, st);
  if (e != 0) return e;
  const int total = B * Ma;
  ng_query_kernel<<<cdiv(total * 32, 256), 256, 0, st>>>(a, Ma, nb.sorted, nb.cell_start, nb.grids, Nb, min_d, arg, total);
  return check_launch("pairwise_min_grid");
}

extern "C" size_t usip_som_assign_grid_scratch_bytes(int B, int M) {
  if (B <= 0 || M <= 0) return 0;
  return (size_t)B * M * sizeof(float4) + (size_t)B * (NG_MAXC + 1) * sizeof(int32_t) + (size_t)B * sizeof(NgGrid) + 64;
}

extern "C" int usip_som_assign_grid_f32(const float* xyz, const float* node, int32_t* min_idx, int32_t* count, void* scratch,
                                        size_t scratch_bytes, int B, int N, int M, void* stream) {
  USIP_REQUIRE(xyz && node && min_idx && scratch && B > 0 && N > 0 && M > 0, "som_assign_grid: bad args");
  USIP_REQUIRE(M <= NGA_MAXM, "som_assign_grid: more than 1024 nodes per cloud (use usip_som_assign_f32)");
  USIP_REQUIRE(scratch_bytes >= usip_som_assign_grid_scratch_bytes(B, M), "som_assign_grid: scratch too small");
  USIP_REQUIRE((reinterpret_cast<uintptr_t>(scratch) & 15) == 0, "som_assign_grid: scratch must be 16-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  float4* sorted = reinterpret_cast<float4*>(scratch);
  int32_t* cell_start = reinterpret_cast<int32_t*>(sorted + (size_t)B * M);
  NgGrid* grids = reinterpret_cast<NgGrid*>(cell_start + (size_t)B * (NG_MAXC + 1));
  grids = reinterpret_cast<NgGrid*>((reinterpret_cast<uintptr_t>(grids) + 15) & ~(uintptr_t)15);
  static bool attr = false;
  const size_t smem = (size_t)(2 * NG_MAXC + 1) * sizeof(int);
  if (!attr) {
    cudaError_t e = cudaFuncSetAttribute(ng_build_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) { set_last_error("som_assign_grid: smem attribute"); return (int)e; }
    attr = true;
  }
  // about two nodes per cell: a 3x3x3 neighbourhood then holds the nearest node of almost every point
  const int max_cells = max(1, min(NGA_MAXC, M / 2));
  ng_build_kernel<<<B, NG_BT, smem, st>>>(node, M, sorted, cell_start, grids, max_cells);
  ng_assign_kernel<<<dim3(cdiv(N, NGA_THREADS), B), NGA_THREADS, 0, st>>>(xyz, N, M, sorted, cell_start, grids, min_idx, count);
  return check_launch("som_assign_grid");
}
