// nngrid.cuh -- the per-cloud cell grid of nngrid.cu, shared with the radius passes of handcrafted.cu.
//
// A grid is cubic cells over the bounding box of a set of queries (at most NG_AXIS per axis and NG_MAXC in all, cells
// widened until both hold), the cloud counting-sorted into it: sorted[b][0..cnt) = (x, y, z, bits(row)) grouped by cell
// (x fastest), cell_start[b][0..ncell] the cells' first slots.  Non-finite rows are left out.
#pragma once
#include "common.cuh"

namespace usip {

constexpr int NG_MAXC = 8192;          // cells per cloud (two int arrays of this size live in shared memory while building)
constexpr int NG_AXIS = 64;            // cells per axis at most

struct NgGrid {
  float ox, oy, oz, h, inv_h;
  int nx, ny, nz;
};

static_assert(sizeof(NgGrid) == 32, "NgGrid is read as two 16-byte words");
__device__ __forceinline__ NgGrid ng_load_grid(const NgGrid* p) {
  const int4 a = __ldg(reinterpret_cast<const int4*>(p)), b = __ldg(reinterpret_cast<const int4*>(p) + 1);
  NgGrid g;
  g.ox = __int_as_float(a.x); g.oy = __int_as_float(a.y); g.oz = __int_as_float(a.z); g.h = __int_as_float(a.w);
  g.inv_h = __int_as_float(b.x); g.nx = b.y; g.ny = b.z; g.nz = b.w;
  return g;
}

__device__ __forceinline__ bool ng_finite3(float x, float y, float z) {
  return (fabsf(x) <= 3.0e38f) && (fabsf(y) <= 3.0e38f) && (fabsf(z) <= 3.0e38f);    // false for NaN and inf
}
__device__ __forceinline__ int ng_cell1(float v, float o, float inv_h, int n) {
  const float t = (v - o) * inv_h;
  return (int)fminf(fmaxf(t, 0.f), (float)(n - 1));              // NaN -> 0 (callers filter non-finite values first)
}

// The multi-CTA build's buffers, carved from one scratch block by ng_build_layout:
// sorted float4 [B][N] | cell_start i32 [B][MAXC+1] | grids [B] (16-byte aligned) | cnt i32 [B][MAXC+1] |
// fill i32 [B][MAXC+1] | cellid i32 [B][N] (the cell of every row, -1 for a non-finite row).
struct NgBuild {
  float4* sorted;
  int32_t* cell_start;
  NgGrid* grids;
  int32_t* cnt;
  int32_t* fill;
  int32_t* cellid;
};

size_t ng_build_bytes(int B, int N);
NgBuild ng_build_layout(void* scratch, int B, int N);
// Grid over the bounding box of qry (B, 3, Ma), cloud pts (B, 3, N) sorted into it: ng_bin_kernel + ng_scatter_kernel
// after one memset.  The order of the entries inside a cell is arbitrary.
int ng_build_multi(const float* qry, int Ma, const float* pts, int N, int B, const NgBuild& s, cudaStream_t st);

}  // namespace usip
