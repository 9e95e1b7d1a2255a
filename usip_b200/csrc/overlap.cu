// overlap.cu -- register2Fragments.m's ratioAligned(1) for many fragment pairs at once: for every point of fragment a,
// is some point of fragment b, mapped into a's frame by the pair's estimate, closer than the radius?  The exact rule
// and the search margin are stated in include/usip_b200.h.
//
// Every fragment is counting-sorted into its own uniform cell grid once per call (a fragment takes part in up to n - 1
// jobs): a bounding box, the cell edge, counts, a per-fragment scan and a scatter.  A query point p of a goes into b's
// frame as q = R^T (p - t) in fp64 and scans every cell that a box of half-width r' around q touches; each candidate's
// b' is recomputed with the job's map and tested exactly.  r' bounds |q - b| for every b that can pass the test, so the
// grid only decides which candidates are looked at, never the answer.
#include <stdlib.h>

#include "common.cuh"

namespace usip {

constexpr int OV_THREADS = 256;
constexpr int OV_SCAN_THREADS = 1024;

struct OvGrid {                 // one fragment's cell grid
  double org[3];                // lower corner of cell (0, 0, 0)
  double h, inv_h;              // cell edge and its reciprocal
  int32_t n[3];                 // cells per axis
  float bmax;                   // max |coordinate| over the finite rows (0 without any)
};

__device__ __forceinline__ bool ov_finite3(float x, float y, float z) {
  return fabsf(x) <= 3.402823466e38f && fabsf(y) <= 3.402823466e38f && fabsf(z) <= 3.402823466e38f;
}

// cell of coordinate v along one axis, clamped into [0, n): monotone in v, so a point inside [lo, hi] lands in a cell
// between those of lo and hi; +-inf clamp to the border cells
__device__ __forceinline__ int ov_axis_cell(double v, double org, double inv_h, int n) {
  const double c = floor(__dmul_rn(__dadd_rn(v, -org), inv_h));
  return c < 0.0 ? 0 : c >= (double)n ? n - 1 : (int)c;
}

__device__ __forceinline__ int64_t ov_cell(const OvGrid& g, double x, double y, double z) {
  const int cx = ov_axis_cell(x, g.org[0], g.inv_h, g.n[0]);
  const int cy = ov_axis_cell(y, g.org[1], g.inv_h, g.n[1]);
  const int cz = ov_axis_cell(z, g.org[2], g.inv_h, g.n[2]);
  return ((int64_t)cz * g.n[1] + cy) * g.n[0] + cx;
}

// grid (chunks, n_frags): per-fragment box of the finite rows as order-preserving words (mins, then maxes)
__global__ void __launch_bounds__(OV_THREADS)
ov_bbox_kernel(const float* __restrict__ xyz, const int64_t* __restrict__ offs, int n_frags, uint32_t* __restrict__ box) {
  const int f = blockIdx.y;
  float lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
  for (int64_t r = offs[f] + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < offs[f + 1];
       r += (int64_t)gridDim.x * blockDim.x) {
    const float x = xyz[3 * r], y = xyz[3 * r + 1], z = xyz[3 * r + 2];
    if (!ov_finite3(x, y, z)) continue;
    lo[0] = fminf(lo[0], x); lo[1] = fminf(lo[1], y); lo[2] = fminf(lo[2], z);
    hi[0] = fmaxf(hi[0], x); hi[1] = fmaxf(hi[1], y); hi[2] = fmaxf(hi[2], z);
  }
#pragma unroll
  for (int c = 0; c < 3; ++c) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      lo[c] = fminf(lo[c], __shfl_xor_sync(0xffffffffu, lo[c], o));
      hi[c] = fmaxf(hi[c], __shfl_xor_sync(0xffffffffu, hi[c], o));
    }
  }
  if ((threadIdx.x & 31) == 0 && lo[0] <= hi[0]) {
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      atomicMin(box + 3 * f + c, f2ord(lo[c]));
      atomicMax(box + 3 * (n_frags + f) + c, f2ord(hi[c]));
    }
  }
}

// one thread per fragment: the cell edge starts at h_min and grows by 1.25 until the grid fits the fragment's cells
__global__ void ov_setup_kernel(const uint32_t* __restrict__ box, const int64_t* __restrict__ cell_off, int n_frags,
                                double h_min, OvGrid* __restrict__ grids) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= n_frags) return;
  const int64_t cap = cell_off[f + 1] - cell_off[f] - 1;
  OvGrid g;
  g.h = h_min; g.n[0] = g.n[1] = g.n[2] = 1; g.org[0] = g.org[1] = g.org[2] = 0.0; g.bmax = 0.f;
  if (box[3 * f] <= box[3 * (n_frags + f)]) {               // any finite row
    double ext[3];
    for (int c = 0; c < 3; ++c) {
      const float lo = ord2f(box[3 * f + c]), hi = ord2f(box[3 * (n_frags + f) + c]);
      g.org[c] = lo;
      ext[c] = (double)hi - (double)lo;
      g.bmax = fmaxf(g.bmax, fmaxf(fabsf(lo), fabsf(hi)));
    }
    for (;;) {
      int64_t tot = 1;
      for (int c = 0; c < 3; ++c) {
        g.n[c] = (int32_t)fmin(floor(ext[c] / g.h) + 1.0, 1048576.0);
        tot *= g.n[c];
      }
      if (tot <= cap) break;
      g.h *= 1.25;
    }
  }
  g.inv_h = 1.0 / g.h;
  grids[f] = g;
}

// grid (chunks, n_frags): rows per cell (count) or each row's place in its cell (scatter)
template <bool SCATTER>
__global__ void __launch_bounds__(OV_THREADS)
ov_bin_kernel(const float* __restrict__ xyz, const int64_t* __restrict__ offs, const int64_t* __restrict__ cell_off,
              const OvGrid* __restrict__ grids, int32_t* __restrict__ cnt, float4* __restrict__ pts) {
  const int f = blockIdx.y;
  const OvGrid g = grids[f];
  int32_t* c = cnt + cell_off[f];
  for (int64_t r = offs[f] + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < offs[f + 1];
       r += (int64_t)gridDim.x * blockDim.x) {
    const float x = xyz[3 * r], y = xyz[3 * r + 1], z = xyz[3 * r + 2];
    if (!ov_finite3(x, y, z)) continue;                     // a non-finite row is never a hit
    const int64_t cell = ov_cell(g, x, y, z);
    if (SCATTER) pts[offs[f] + atomicAdd(c + cell, 1)] = make_float4(x, y, z, 0.f);
    else atomicAdd(c + cell, 1);
  }
}

// one CTA per fragment: exclusive scan of its cells + 1 counts in place.  After the scatter, entry c holds the end of
// cell c (the start of c + 1), so cell c's rows are [c ? cnt[c - 1] : 0, cnt[c]).
__global__ void __launch_bounds__(OV_SCAN_THREADS)
ov_scan_kernel(const int64_t* __restrict__ cell_off, const OvGrid* __restrict__ grids, int32_t* __restrict__ cnt) {
  __shared__ int32_t wsum[32];
  __shared__ int32_t carry_s;
  const int f = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const OvGrid g = grids[f];
  const int64_t n = (int64_t)g.n[0] * g.n[1] * g.n[2] + 1;
  int32_t* c = cnt + cell_off[f];
  if (tid == 0) carry_s = 0;
  __syncthreads();
  for (int64_t base = 0; base < n; base += OV_SCAN_THREADS) {
    const int64_t i = base + tid;
    const int32_t v = i < n ? c[i] : 0;
    int32_t x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int32_t y = __shfl_up_sync(0xffffffffu, x, o);
      if (lane >= o) x += y;
    }
    if (lane == 31) wsum[warp] = x;
    __syncthreads();
    if (warp == 0) {
      int32_t w = wsum[lane];
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int32_t y = __shfl_up_sync(0xffffffffu, w, o);
        if (lane >= o) w += y;
      }
      wsum[lane] = w;
    }
    __syncthreads();
    const int32_t excl = carry_s + (warp ? wsum[warp - 1] : 0) + x - v;
    if (i < n) c[i] = excl;
    __syncthreads();
    if (tid == OV_SCAN_THREADS - 1) carry_s = excl + v;
    __syncthreads();
  }
}

// blockIdx.x -> job j (the last with blk[j] <= blockIdx.x) and a 256-row slice of fragment a; hits[j] += the slice's
// hits
__global__ void __launch_bounds__(OV_THREADS)
ov_query_kernel(const float* __restrict__ xyz, const int64_t* __restrict__ offs, const int64_t* __restrict__ cell_off,
                const OvGrid* __restrict__ grids, const int32_t* __restrict__ cnt, const float4* __restrict__ pts,
                const int32_t* __restrict__ jobs, const int64_t* __restrict__ blk, int J, const double* __restrict__ Rt,
                float radius, float t_lim, int32_t* __restrict__ hits) {
  __shared__ double sRt[12];
  __shared__ double s_r0, s_tmax;
  __shared__ int32_t s_job;
  __shared__ int32_t s_sum[OV_THREADS / 32];
  const int tid = threadIdx.x;
  if (tid == 0) {
    int lo = 0, hi = J;
    while (hi - lo > 1) {
      const int mid = (lo + hi) >> 1;
      if (blk[mid] <= (int64_t)blockIdx.x) lo = mid; else hi = mid;
    }
    s_job = lo;
  }
  __syncthreads();
  const int j = s_job;
  const int fa = jobs[2 * j], fb = jobs[2 * j + 1];
  const OvGrid g = grids[fb];
  if (tid < 12) sRt[tid] = Rt[12 * (int64_t)j + tid];
  __syncthreads();
  if (tid == 0) {
    // delta = max |(R^T R - I)_ik|; B = max_i sum_k |R_ik| bmax + |t_i| bounds every |b'_i| (see the header)
    double delta = 0.0, B = 0.0, tmax = 0.0;
    for (int i = 0; i < 3; ++i) {
      for (int k = 0; k < 3; ++k) {
        double s = 0.0;
        for (int r = 0; r < 3; ++r) s += sRt[4 * r + i] * sRt[4 * r + k];
        delta = fmax(delta, fabs(s - (i == k ? 1.0 : 0.0)));
      }
      const double row = fabs(sRt[4 * i]) + fabs(sRt[4 * i + 1]) + fabs(sRt[4 * i + 2]);
      B = fmax(B, row * (double)g.bmax + fabs(sRt[4 * i + 3]));
      tmax = fmax(tmax, fabs(sRt[4 * i + 3]));
    }
    delta += 0x1p-40;
    const double D = (double)radius * (1.0 + 0x1p-20) + 0x1p-23 * B + 1e-30;
    s_r0 = D * (1.0 + 2.0 * delta) + 6.0 * delta * (double)g.bmax;   // NaN when Rt is not finite
    s_tmax = tmax;
  }
  __syncthreads();
  const int64_t row = offs[fa] + ((int64_t)blockIdx.x - blk[j]) * OV_THREADS + tid;
  int hit = 0;
  if (row < offs[fa + 1]) {
    const float px = xyz[3 * row], py = xyz[3 * row + 1], pz = xyz[3 * row + 2];
    if (ov_finite3(px, py, pz)) {
      const double dx = __dadd_rn((double)px, -sRt[3]), dy = __dadd_rn((double)py, -sRt[7]),
                   dz = __dadd_rn((double)pz, -sRt[11]);
      double q[3];
#pragma unroll
      for (int c = 0; c < 3; ++c)
        q[c] = __dadd_rn(__dadd_rn(__dmul_rn(sRt[c], dx), __dmul_rn(sRt[4 + c], dy)), __dmul_rn(sRt[8 + c], dz));
      const double pm = fmax(fmax(fabs((double)px), fabs((double)py)), fabs((double)pz));
      const double r = s_r0 + 0x1p-40 * (pm + s_tmax + (double)g.bmax);
      int lo[3], hi[3];
      const bool all = !(fabs(r) <= 1.7e308) || !(fabs(q[0]) + fabs(q[1]) + fabs(q[2]) <= 1.7e308);
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        lo[c] = all ? 0 : ov_axis_cell(__dadd_rn(q[c], -r), g.org[c], g.inv_h, g.n[c]);
        hi[c] = all ? g.n[c] - 1 : ov_axis_cell(__dadd_rn(q[c], r), g.org[c], g.inv_h, g.n[c]);
      }
      const int32_t* cs = cnt + cell_off[fb];
      const float4* pb = pts + offs[fb];
      for (int cz = lo[2]; cz <= hi[2] && !hit; ++cz)
        for (int cy = lo[1]; cy <= hi[1] && !hit; ++cy) {
          const int64_t c0 = ((int64_t)cz * g.n[1] + cy) * g.n[0];
          const int32_t k0 = (c0 + lo[0]) ? cs[c0 + lo[0] - 1] : 0, k1 = cs[c0 + hi[0]];
          for (int k = k0; k < k1; ++k) {
            const float4 b = pb[k];
            double x = b.x, y = b.y, z = b.z;
            reg_map(sRt, x, y, z);
            if (sqdist_rn(px, py, pz, __double2float_rn(x), __double2float_rn(y), __double2float_rn(z)) <= t_lim) {
              hit = 1;
              break;
            }
          }
        }
    }
  }
  const unsigned any = __ballot_sync(0xffffffffu, hit);
  if ((tid & 31) == 0) s_sum[tid >> 5] = __popc(any);
  __syncthreads();
  if (tid == 0) {
    int s = 0;
    for (int w = 0; w < OV_THREADS / 32; ++w) s += s_sum[w];
    if (s) atomicAdd(hits + j, s);
  }
}

// the largest fp32 t with sqrtf(t) < radius (radius > 0 and finite): d2 <= t  <=>  sqrtf(d2) < radius
float ov_strict_tlim_host(float radius) {
  float t = radius * radius;
  while (t > 0.f && !(sqrtf(t) < radius)) t = nextafterf(t, 0.f);
  for (;;) {
    const float up = nextafterf(t, INFINITY);
    if (isinf(up) || !(sqrtf(up) < radius)) break;
    t = up;
  }
  return t;
}

struct OvLayout {               // byte offsets into the scratch, each 16-byte aligned
  size_t offs, cell_off, blk, jobs, box, grids, cnt, pts, total;
};

inline size_t ov_align(size_t b) { return (b + 15) & ~(size_t)15; }

OvLayout ov_layout(int64_t total_rows, int n_frags, int J) {
  OvLayout L;
  size_t at = 0;
  L.offs = at;     at += ov_align(sizeof(int64_t) * (n_frags + 1));
  L.cell_off = at; at += ov_align(sizeof(int64_t) * (n_frags + 1));
  L.blk = at;      at += ov_align(sizeof(int64_t) * (J + 1));
  L.jobs = at;     at += ov_align(sizeof(int32_t) * 2 * (size_t)J);
  L.box = at;      at += ov_align(sizeof(uint32_t) * 6 * (size_t)n_frags);
  L.grids = at;    at += ov_align(sizeof(OvGrid) * (size_t)n_frags);
  L.cnt = at;      at += ov_align(sizeof(int32_t) * (size_t)(2 * total_rows + 65 * (int64_t)n_frags));
  L.pts = at;      at += ov_align(sizeof(float4) * (size_t)total_rows);
  L.total = at;
  return L;
}

}  // namespace usip

using namespace usip;

extern "C" size_t usip_fragment_overlap_scratch_bytes(int64_t total_rows, int n_frags, int J) {
  if (total_rows < 0 || n_frags < 1 || J < 1) return 0;
  return ov_layout(total_rows, n_frags, J).total;
}

extern "C" int usip_fragment_overlap_f32(const float* xyz, const int64_t* offsets, int n_frags, const int32_t* jobs,
                                         const double* Rt, int J, float radius, void* scratch, size_t scratch_bytes,
                                         int32_t* hits, void* stream) {
  USIP_REQUIRE(xyz && offsets && jobs && Rt && scratch && hits, "fragment_overlap: null pointer");
  USIP_REQUIRE(n_frags >= 1 && J >= 1, "fragment_overlap: need at least one fragment and one job");
  USIP_REQUIRE(radius > 0.f && radius <= 3.4e38f, "fragment_overlap: radius must be > 0 and finite");
  USIP_REQUIRE(n_frags <= 65535, "fragment_overlap: at most 65535 fragments per call");
  USIP_REQUIRE(offsets[0] == 0, "fragment_overlap: offsets[0] must be 0");
  int64_t max_rows = 0;
  for (int f = 0; f < n_frags; ++f) {
    const int64_t n = offsets[f + 1] - offsets[f];
    USIP_REQUIRE(n >= 1, "fragment_overlap: a fragment has no rows");
    USIP_REQUIRE(n <= USIP_OVERLAP_MAX_ROWS, "fragment_overlap: a fragment has more than USIP_OVERLAP_MAX_ROWS rows");
    max_rows = n > max_rows ? n : max_rows;
  }
  const int64_t total = offsets[n_frags];
  const OvLayout L = ov_layout(total, n_frags, J);
  USIP_REQUIRE(((uintptr_t)scratch & 15) == 0, "fragment_overlap: scratch must be 16-byte aligned");
  USIP_REQUIRE(scratch_bytes >= L.total, "fragment_overlap: scratch smaller than usip_fragment_overlap_scratch_bytes");
  // host metadata: offsets, cell offsets (2 rows + 65 per fragment), per-job first block, jobs
  char* s = (char*)scratch;
  const size_t meta = L.box;
  char* h = (char*)calloc(meta, 1);
  USIP_REQUIRE(h, "fragment_overlap: host allocation failed");
  int64_t* h_offs = (int64_t*)(h + L.offs);
  int64_t* h_cell = (int64_t*)(h + L.cell_off);
  int64_t* h_blk = (int64_t*)(h + L.blk);
  int32_t* h_jobs = (int32_t*)(h + L.jobs);
  h_cell[0] = 0;
  for (int f = 0; f <= n_frags; ++f) h_offs[f] = offsets[f];
  for (int f = 0; f < n_frags; ++f) h_cell[f + 1] = h_cell[f] + 2 * (offsets[f + 1] - offsets[f]) + 65;
  h_blk[0] = 0;
  for (int j = 0; j < J; ++j) {
    const int a = jobs[2 * j], b = jobs[2 * j + 1];
    if (a < 0 || a >= n_frags || b < 0 || b >= n_frags) { free(h); return fail("fragment_overlap: a job names a fragment out of range"); }
    h_jobs[2 * j] = a; h_jobs[2 * j + 1] = b;
    h_blk[j + 1] = h_blk[j] + cdiv64(offsets[a + 1] - offsets[a], OV_THREADS);
  }
  const int64_t blocks = h_blk[J];
  if (blocks > 0x7fffffffll) { free(h); return fail("fragment_overlap: more query blocks than one launch holds"); }
  cudaStream_t st = (cudaStream_t)stream;
  cudaError_t e = cudaMemcpyAsync(s, h, meta, cudaMemcpyHostToDevice, st);     // pageable: staged before returning
  free(h);
  if (e != cudaSuccess) { set_last_error("fragment_overlap: metadata copy"); return (int)e; }
  if ((e = cudaMemsetAsync(s + L.box, 0xff, sizeof(uint32_t) * 3 * (size_t)n_frags, st)) != cudaSuccess ||
      (e = cudaMemsetAsync(s + L.box + sizeof(uint32_t) * 3 * (size_t)n_frags, 0, sizeof(uint32_t) * 3 * (size_t)n_frags,
                           st)) != cudaSuccess ||
      (e = cudaMemsetAsync(s + L.cnt, 0, L.pts - L.cnt, st)) != cudaSuccess ||
      (e = cudaMemsetAsync(hits, 0, sizeof(int32_t) * (size_t)J, st)) != cudaSuccess) {
    set_last_error("fragment_overlap: memset");
    return (int)e;
  }
  const int64_t* d_offs = (const int64_t*)(s + L.offs);
  const int64_t* d_cell = (const int64_t*)(s + L.cell_off);
  OvGrid* grids = (OvGrid*)(s + L.grids);
  int32_t* cnt = (int32_t*)(s + L.cnt);
  float4* pts = (float4*)(s + L.pts);
  const int64_t chunks = cdiv64(max_rows, OV_THREADS * 8);
  const dim3 rows_grid((unsigned)(chunks < 256 ? chunks : 256), (unsigned)n_frags);
  ov_bbox_kernel<<<rows_grid, OV_THREADS, 0, st>>>(xyz, d_offs, n_frags, (uint32_t*)(s + L.box));
  ov_setup_kernel<<<cdiv(n_frags, 128), 128, 0, st>>>((const uint32_t*)(s + L.box), d_cell, n_frags,
                                                      (double)radius * 1.01, grids);
  ov_bin_kernel<false><<<rows_grid, OV_THREADS, 0, st>>>(xyz, d_offs, d_cell, grids, cnt, pts);
  ov_scan_kernel<<<n_frags, OV_SCAN_THREADS, 0, st>>>(d_cell, grids, cnt);
  ov_bin_kernel<true><<<rows_grid, OV_THREADS, 0, st>>>(xyz, d_offs, d_cell, grids, cnt, pts);
  ov_query_kernel<<<(unsigned)blocks, OV_THREADS, 0, st>>>(xyz, d_offs, d_cell, grids, cnt, pts,
                                                           (const int32_t*)(s + L.jobs), (const int64_t*)(s + L.blk), J,
                                                           Rt, radius, ov_strict_tlim_host(radius), hits);
  return check_launch("ov_query_kernel");
}
