// ballgroup.cu -- fused ball query + group (models/networks.py:355-373 + ball_query_ext/ball_query_cuda.cu:10-49): two
// launches chained by programmatic dependent launch, candidate tiles staged by tensor-map TMA in shared memory.
//
//   bx_build_kernel  every CTA derives the same 2-D bucket grid from the CENTRES of its cloud (bounding box of the
//                    keypoints grown by two cells; the axis with the smallest extent is not binned; cell size h >= 1.001 r,
//                    fixed row pitch), then drops its points into fixed-capacity buckets: slot = atomicAdd(count[cell]);
//                    record (x,y,z,index | f0..f3) -> bucket[cell][slot], or -> the cloud's overflow list when the bucket
//                    is full.  No histogram, no scan, no second pass: points farther than a cell from every centre are
//                    dropped on the spot.  Four points per thread, their four atomics in flight together.
//   bx_query_kernel  one warp per keypoint: the 3 x 3 neighbouring buckets are a 768-byte x 3-row box of the cloud's bucket
//                    plane (fixed pitch of 128 cells); one elected lane fetches the box with ONE tensor-map TMA
//                    (cp.async.bulk.tensor.3d -> UTMALDG, mbarrier complete_tx) while nine lanes read the nine fill counts;
//                    warp-ballot radius test on the staged records; hits are ranked by point index (the reference keeps the
//                    FIRST K hits in index order) and index, gathered record and decentred group are written in one pass of
//                    full 128-byte lines.  The last CTA of a cloud to finish clears the counts again, so the scratch is left
//                    as it was found: all-zero counters.
//
// Exactness: d^2 with the reference's fp32 op order against t_max (ballquery.cu), cell size h >= 1.001 r so every point
// within r of a centre lies in the 3 x 3 block around the centre's cell; clouds whose overflow list is full, balls with
// more than 64 hits, K > 64 and non-finite radii take the reference's own in-order scan (bit-identical by construction).
#include "tc_common.cuh"
#include <cstdlib>

namespace usip {

constexpr int BX_CAP = 8;                 // records per bucket: 8 x 32 B = 256 B, a 3-bucket row is one 768-byte bulk copy
constexpr int BX_PITCH = 128;             // cells per row of the bucket plane (fixed, so ONE tensor map describes every cloud)
constexpr int BX_ROWS = 128;              // rows of the bucket plane
constexpr int BX_MAX_CELLS = BX_PITCH * BX_ROWS;   // per cloud -> 4 MB of buckets
constexpr int BX_OVF = 4096;              // overflow records per cloud before the cloud falls back to the in-order scan
constexpr int BX_HITS = 64;               // hits kept per keypoint before the in-order fallback (= max K of the fast path)
constexpr int BX_CHUNK = 1024;            // points per CTA in the build kernel (4 per thread: 4 atomics in flight)

struct BxGrid { float o0, o1, inv_h; int n0, n1, a0, a1, ok; };            // 32 bytes

struct BxScratch {
  BxGrid* grids; int32_t* counts; int32_t* ovf_cnt; int32_t* done; float4* buckets; float4* ovf; size_t total;
  __host__ __device__ static size_t align(size_t x) { return (x + 255) & ~(size_t)255; }
  __host__ BxScratch(void* base, int B) {
    size_t off = 0;
    auto take = [&](size_t bytes) { size_t o = off; off += align(bytes); return o; };
    const size_t o_c = take(sizeof(int32_t) * (size_t)B * BX_MAX_CELLS);   // zero-state region first (one memset)
    const size_t o_o = take(sizeof(int32_t) * B), o_d = take(sizeof(int32_t) * B);
    const size_t zero_end = off;
    const size_t o_g = take(sizeof(BxGrid) * B);
    const size_t o_b = take(sizeof(float4) * 2 * (size_t)B * BX_MAX_CELLS * BX_CAP);
    const size_t o_v = take(sizeof(float4) * 2 * (size_t)B * BX_OVF);
    total = off; zero_bytes = zero_end;
    char* p = (char*)base;
    counts = (int32_t*)(p + o_c); ovf_cnt = (int32_t*)(p + o_o); done = (int32_t*)(p + o_d); grids = (BxGrid*)(p + o_g);
    buckets = (float4*)(p + o_b); ovf = (float4*)(p + o_v);
  }
  size_t zero_bytes;
};

__device__ __forceinline__ float bx_axis(float x, float y, float z, int a) { return a == 0 ? x : (a == 1 ? y : z); }

// Bounding box of the finite centres of one cloud -> bucket grid.  Every CTA computes the same values (same operations
// in the same order on the same data), so no launch and no memory round trip is spent on publishing the grid.
__device__ BxGrid bx_make_grid(const float* __restrict__ cp, int M, float radius, float (*red)[8]) {
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5, nw = blockDim.x >> 5;
  float lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
  for (int m = tid; m < M; m += blockDim.x) {
    const float c[3] = {cp[m], cp[M + m], cp[2 * M + m]};
    if (fabsf(c[0]) <= 1e30f && fabsf(c[1]) <= 1e30f && fabsf(c[2]) <= 1e30f) {
#pragma unroll
      for (int a = 0; a < 3; ++a) { lo[a] = fminf(lo[a], c[a]); hi[a] = fmaxf(hi[a], c[a]); }
    }
  }
#pragma unroll
  for (int a = 0; a < 3; ++a) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      lo[a] = fminf(lo[a], __shfl_xor_sync(0xffffffffu, lo[a], o));
      hi[a] = fmaxf(hi[a], __shfl_xor_sync(0xffffffffu, hi[a], o));
    }
    if (lane == 0) { red[a][w] = lo[a]; red[3 + a][w] = hi[a]; }
  }
  __syncthreads();
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    lo[a] = INFINITY; hi[a] = -INFINITY;
    for (int i = 0; i < nw; ++i) { lo[a] = fminf(lo[a], red[a][i]); hi[a] = fmaxf(hi[a], red[3 + a][i]); }
  }
  BxGrid g;
  g.ok = (radius >= 0.f) && (radius <= 1e30f) && (lo[0] <= hi[0]);
  const float e[3] = {hi[0] - lo[0], hi[1] - lo[1], hi[2] - lo[2]};
  int drop = 0;                                               // the axis with the smallest extent is not binned
  if (e[1] < e[drop]) drop = 1;
  if (e[2] < e[drop]) drop = 2;
  g.a0 = drop == 0 ? 1 : 0; g.a1 = drop == 2 ? 1 : 2;
  const float e0 = bx_axis(e[0], e[1], e[2], g.a0), e1 = bx_axis(e[0], e[1], e[2], g.a1);       // (selects, no local arrays)
  const float lo0 = bx_axis(lo[0], lo[1], lo[2], g.a0), lo1 = bx_axis(lo[0], lo[1], lo[2], g.a1);
  float h = fmaxf(radius * 1.001f, 1e-6f);
  int n0 = 1, n1 = 1;
  if (g.ok) {
    for (int it = 0; it < 96; ++it) {
      // two margin cells on either side: a centre's cell index stays in [1, n-2] whatever the last-bit rounding of
      // (c - o) * inv_h does, so its 3 x 3 block never leaves the grid
      n0 = (int)fminf(floorf(e0 / h), 1e6f) + 5; n1 = (int)fminf(floorf(e1 / h), 1e6f) + 5;
      if (n0 <= BX_PITCH && n1 <= BX_ROWS) break;
      h *= 1.26f;
    }
    if (n0 > BX_PITCH || n1 > BX_ROWS) g.ok = 0;
  }
  g.o0 = lo0 - 2.f * h; g.o1 = lo1 - 2.f * h; g.inv_h = 1.0f / h; g.n0 = n0; g.n1 = n1;
  return g;
}

__global__ void __launch_bounds__(256)
bx_build_kernel(const float* __restrict__ xyz, const float* __restrict__ feat, const float* __restrict__ centers,
                float radius, BxGrid* __restrict__ grids, int32_t* __restrict__ counts, int32_t* __restrict__ ovf_cnt,
                float4* __restrict__ buckets, float4* __restrict__ ovf, int S, int N, int M) {
  __shared__ float red[6][8];
  const int b = blockIdx.y, tid = threadIdx.x;
  const float* p = xyz + (size_t)b * 3 * N;
  // the point loads do not depend on the grid: issue them first, the centre reduction runs in their shadow.  Everything
  // is indexed by compile-time constants (fully unrolled): no local-memory arrays.
  float px[4], py[4], pz[4], pf[4][4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int n = blockIdx.x * BX_CHUNK + j * 256 + tid;
    const bool in = n < N;
    px[j] = in ? __ldg(p + n) : NAN; py[j] = in ? __ldg(p + N + n) : NAN; pz[j] = in ? __ldg(p + 2 * N + n) : NAN;
#pragma unroll
    for (int c = 0; c < 4; ++c) pf[j][c] = (in && c < S) ? __ldg(feat + ((size_t)b * S + c) * N + n) : 0.f;
  }
  const BxGrid g = bx_make_grid(centers + (size_t)b * 3 * M, M, radius, red);
  if (blockIdx.x == 0 && tid == 0) grids[b] = g;
  // let the query kernel's CTAs start (they wait for this grid's completion before touching the buckets)
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  if (!g.ok) return;
  int32_t* cnt = counts + (size_t)b * BX_MAX_CELLS;
  float4* bk = buckets + (size_t)b * BX_MAX_CELLS * BX_CAP * 2;
  // all four fill-count atomics are issued before any of their results is used (four L2 round trips in flight)
  int cell[4], slot[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float x = px[j], y = py[j], z = pz[j];
    cell[j] = -1;
    if (fabsf(x) <= 1e30f && fabsf(y) <= 1e30f && fabsf(z) <= 1e30f) {            // non-finite (and n >= N): never within a finite radius
      const float f0 = floorf((bx_axis(x, y, z, g.a0) - g.o0) * g.inv_h), f1 = floorf((bx_axis(x, y, z, g.a1) - g.o1) * g.inv_h);
      if (f0 >= 0.f && f0 < (float)g.n0 && f1 >= 0.f && f1 < (float)g.n1) cell[j] = (int)f1 * BX_PITCH + (int)f0;   // else: farther than a cell from every centre
    }
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) slot[j] = cell[j] >= 0 ? atomicAdd(cnt + cell[j], 1) : 0;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    if (cell[j] < 0) continue;
    const int n = blockIdx.x * BX_CHUNK + j * 256 + tid;
    float4* dst;
    if (slot[j] < BX_CAP) {
      dst = bk + ((size_t)cell[j] * BX_CAP + slot[j]) * 2;
    } else {
      const int o = atomicAdd(ovf_cnt + b, 1);
      if (o >= BX_OVF) continue;                             // the query sees ovf_cnt > BX_OVF and scans the cloud in order
      dst = ovf + ((size_t)b * BX_OVF + o) * 2;
    }
    dst[0] = make_float4(px[j], py[j], pz[j], __int_as_float(n));
    dst[1] = make_float4(pf[j][0], pf[j][1], pf[j][2], pf[j][3]);
  }
}

__global__ void __launch_bounds__(256)
bx_query_kernel(const __grid_constant__ CUtensorMap tmap, const float* __restrict__ xyz, const float* __restrict__ feat,
                const float* __restrict__ centers,
                const BxGrid* __restrict__ grids, int32_t* __restrict__ counts, int32_t* __restrict__ ovf_cnt,
                int32_t* __restrict__ done, const float4* __restrict__ buckets, const float4* __restrict__ ovf,
                float t_max, int32_t* __restrict__ out_idx, float* __restrict__ out_group, float* __restrict__ out_rows,
                int ld_rows, int B, int S, int N, int M, int K, int ctas_per_cloud) {
  __shared__ __align__(128) float4 stage[8][9 * BX_CAP * 2];       // 8 warps x 2304 B: the 3 x 3 buckets of the warp's keypoint
  __shared__ __align__(16) float4 hrec[8][2][BX_HITS];            // the hits' records (x,y,z,n | f0..f3)
  __shared__ int hidx[8][2][BX_HITS];                             // point indices in discovery order; discovery positions in index order
  __shared__ __align__(8) uint64_t mbar[8];
  __shared__ int s_last;
  const int wib = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // grid = (ceil(M / 8), B): CTAs never straddle clouds, so the arrival counter below is per cloud
  const int b = blockIdx.y, m = blockIdx.x * 8 + wib;
  const bool active = m < M;
  const int w = b * M + m;
  const float* cp = centers + (size_t)b * 3 * M;
  float cx = 0.f, cy = 0.f, cz = 0.f;
  if (active) { cx = __ldg(cp + m); cy = __ldg(cp + M + m); cz = __ldg(cp + 2 * M + m); }   // inputs: legal before the dependency wait
  const uint32_t bar = smem_u32(&mbar[wib]);
  if (lane == 0) { mbar_init(bar, 1); fence_barrier_init(); }
  __syncwarp();
  asm volatile("griddepcontrol.wait;" ::: "memory");                // the build grid has completed and its writes are visible
  const BxGrid g = grids[b];                    // L1-cached: 8 warps x ~14 CTAs per SM read the same 32 bytes (measured: the
                                                // L2-only load cost 4 us on the whole kernel)
  const float* p = xyz + (size_t)b * 3 * N;
  int32_t* cnt = counts + (size_t)b * BX_MAX_CELLS;
  const unsigned lt = (1u << lane) - 1u;
  const int C = 3 + S;
  int nh = 0;
  bool brute = !g.ok || K > BX_HITS;
  int32_t* o = out_idx + (size_t)w * K;
  int* hn = hidx[wib][0]; int* sl = hidx[wib][1];
  float4* h0 = hrec[wib][0]; float4* h1 = hrec[wib][1];
  if (active) {
    const int novf = __ldg(ovf_cnt + b);
    if (novf > BX_OVF) brute = true;
    const bool cfin = fabsf(cx) <= 1e30f && fabsf(cy) <= 1e30f && fabsf(cz) <= 1e30f;
    if (!brute && cfin) {
      // finite centres lie in cells [1, n-2] (bx_make_grid): the 3 x 3 block never leaves the grid; the clamp only
      // guards the address arithmetic
      const int k0 = min(max((int)floorf((bx_axis(cx, cy, cz, g.a0) - g.o0) * g.inv_h), 1), g.n0 - 2);
      const int k1 = min(max((int)floorf((bx_axis(cx, cy, cz, g.a1) - g.o1) * g.inv_h), 1), g.n1 - 2);
      const int base = (k1 - 1) * BX_PITCH + (k0 - 1);
      float4* st = stage[wib];
      if (lane == 0) {
        // box = 3 buckets (192 floats) x 3 rows of cloud b's bucket plane, landing as three consecutive 768-byte rows
        mbar_arrive_expect_tx(bar, 3 * 3 * BX_CAP * 32);
        asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];"
                     ::"r"(smem_u32(st)), "l"(&tmap), "r"((k0 - 1) * (BX_CAP * 8)), "r"(k1 - 1), "r"(b), "r"(bar) : "memory");
      }
      int fill = 0;                                               // lanes 0..8: fill count of bucket (lane / 3, lane % 3)
      const int l3 = (lane * 11) >> 5;                          // lane / 3 for lane < 9
      if (lane < 9) fill = __ldcg(cnt + base + l3 * BX_PITCH + (lane - 3 * l3));
      const unsigned over = __ballot_sync(0xffffffffu, fill > BX_CAP);
      mbar_wait_sleep(bar, 0);
      // 72 slots, 32 per pass: slot s belongs to bucket s / 8
      for (int s0 = 0; s0 < 9 * BX_CAP && !brute; s0 += 32) {
        const int s = s0 + lane;
        const int f = __shfl_sync(0xffffffffu, fill, (s < 9 * BX_CAP ? s : 0) / BX_CAP);
        bool hit = false;
        float4 q = make_float4(0.f, 0.f, 0.f, 0.f), qf = q;
        if (s < 9 * BX_CAP && (s % BX_CAP) < f) {
          q = st[2 * s]; qf = st[2 * s + 1];
          hit = sqdist_rn(cx, cy, cz, q.x, q.y, q.z) <= t_max;
        }
        const unsigned bal = __ballot_sync(0xffffffffu, hit);
        if (bal) {
          const int pos = nh + __popc(bal & lt);
          if (hit && pos < BX_HITS) { hn[pos] = __float_as_int(q.w); h0[pos] = q; h1[pos] = qf; }
          nh += __popc(bal);
          if (nh > BX_HITS) brute = true;
        }
      }
      if (over && !brute) {
        // a neighbouring bucket overflowed: its surplus records sit in the cloud's (short) overflow list
        const float4* ov = ovf + (size_t)b * BX_OVF * 2;
        for (int s0 = 0; s0 < novf && !brute; s0 += 32) {
          const int s = s0 + lane;
          bool hit = false;
          float4 q = make_float4(0.f, 0.f, 0.f, 0.f), qf = q;
          if (s < novf) { q = __ldcg(ov + 2 * s); qf = __ldcg(ov + 2 * s + 1); hit = sqdist_rn(cx, cy, cz, q.x, q.y, q.z) <= t_max; }
          const unsigned bal = __ballot_sync(0xffffffffu, hit);
          if (bal) {
            const int pos = nh + __popc(bal & lt);
            if (hit && pos < BX_HITS) { hn[pos] = __float_as_int(q.w); h0[pos] = q; h1[pos] = qf; }
            nh += __popc(bal);
            if (nh > BX_HITS) brute = true;
          }
        }
      }
    }
    __syncwarp();
    if (brute) {
      // the reference loop itself: in-order scan with early exit (dense balls, degenerate grids, K > 64, flooded overflow)
      nh = 0;
      for (int n0 = 0; n0 < N && nh < K; n0 += 32) {
        const int n = n0 + lane;
        const bool hit = (n < N) && (sqdist_rn(cx, cy, cz, __ldg(p + n), __ldg(p + N + n), __ldg(p + 2 * N + n)) <= t_max);
        const unsigned bal = __ballot_sync(0xffffffffu, hit);
        if (bal) {
          const int pos = nh + __popc(bal & lt);
          if (hit && pos < K) o[pos] = n;
          nh += __popc(bal);
        }
      }
      __syncwarp();
    } else {
      // order by point index: rank = number of hits with a smaller index (indices are distinct)
      for (int i = lane; i < nh; i += 32) {
        const int mine = hn[i];
        int rk = 0;
        for (int j = 0; j < nh; ++j) rk += hn[j] < mine ? 1 : 0;
        sl[rk] = i;
      }
      __syncwarp();
    }
    // out[k] = hits[k % u] (first u in index order, then the cyclic pad of ball_query_cuda.cu:40-46); no hit -> point 0
    const int u = min(nh, K);
    const float ru = u > 1 ? __frcp_rn((float)u) : 0.f;        // k, u <= 64: floor((k + 0.5) / u) is exact in fp32
    const float* pfeat = feat + (size_t)b * S * N;
    for (int k = lane; k < K; k += 32) {
      const int e = u > 1 ? (k - u * (int)(((float)k + 0.5f) * ru)) : 0;    // k % u
      int n = 0;
      float v[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
      if (!brute && u > 0) {
        const float4 r0 = h0[sl[e]], r1 = h1[sl[e]];
        n = __float_as_int(r0.w);
        v[0] = r0.x - cx; v[1] = r0.y - cy; v[2] = r0.z - cz; v[3] = r1.x; v[4] = r1.y; v[5] = r1.z; v[6] = r1.w;   // networks.py:373
      } else {
        n = u > 0 ? o[e] : 0;
        if (out_group || out_rows) {
          v[0] = __ldg(p + n) - cx; v[1] = __ldg(p + N + n) - cy; v[2] = __ldg(p + 2 * N + n) - cz;
#pragma unroll
          for (int c = 0; c < 4; ++c) if (c < S) v[3 + c] = __ldg(pfeat + (size_t)c * N + n);
        }
      }
      if (!brute || k >= u) o[k] = n;
      if (out_group) {
        float* gp = out_group + ((size_t)b * C * M + m) * K + k;
#pragma unroll
        for (int c = 0; c < 7; ++c) if (c < C) __stcs(gp + (size_t)c * M * K, v[c]);      // streaming: written once, read by the next op
      }
      if (out_rows) {
        float* rowp = out_rows + ((size_t)w * K + k) * ld_rows;
        if (ld_rows == 8) {
          __stcs(reinterpret_cast<float4*>(rowp), make_float4(v[0], v[1], v[2], v[3]));
          __stcs(reinterpret_cast<float4*>(rowp) + 1, make_float4(v[4], v[5], v[6], v[7]));
        } else {
#pragma unroll
          for (int c = 0; c < 8; ++c) if (c < ld_rows) rowp[c] = c < C ? v[c] : 0.f;
          for (int c = 8; c < ld_rows; ++c) rowp[c] = 0.f;
        }
      }
    }
  }
  // restore the zero state: the last CTA of this cloud clears the fill counts (all other CTAs have finished reading them)
  __syncthreads();
  if (threadIdx.x == 0) { __threadfence(); s_last = atomicAdd(done + b, 1) == ctas_per_cloud - 1; }
  __syncthreads();
  if (s_last) {
    const int cells = g.ok ? g.n1 * BX_PITCH : 0;              // rows 0..n1-1 of the fixed-pitch plane
    for (int i = threadIdx.x; i < cells / 4; i += blockDim.x) reinterpret_cast<int4*>(cnt)[i] = make_int4(0, 0, 0, 0);
    if (threadIdx.x == 0) { ovf_cnt[b] = 0; done[b] = 0; }
  }
}

float radius_to_tmax_host(float radius);          // ballquery.cu

// Tensor map of the bucket planes: 3-D tensor [B clouds][BX_ROWS rows][BX_PITCH cells x 64 floats], box = 3 cells x 3 rows.
static int bx_tensor_map(CUtensorMap* tm, float4* buckets, int B) {
  const cuuint64_t dims[3] = {(cuuint64_t)BX_PITCH * BX_CAP * 8, (cuuint64_t)BX_ROWS, (cuuint64_t)B};
  const cuuint64_t strides[2] = {(cuuint64_t)BX_PITCH * BX_CAP * 32, (cuuint64_t)BX_MAX_CELLS * BX_CAP * 32};   // bytes, dims 1..2
  const cuuint32_t box[3] = {3 * BX_CAP * 8, 3, 1};
  const cuuint32_t estr[3] = {1, 1, 1};
  return encode_tensor_map_tiled(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, buckets, dims, strides, box, estr,
                                 CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_NONE, "ball_group: bucket tensor map");
}

}  // namespace usip

using namespace usip;

extern "C" int64_t usip_ball_group_scratch_bytes(int B, int S, int N, int M, int K) {
  (void)S; (void)N; (void)M; (void)K;
  BxScratch sc(nullptr, B);
  return (int64_t)sc.total + 256;
}

extern "C" int usip_ball_group_scratch_init(void* scratch, int64_t scratch_bytes, int B, void* stream) {
  USIP_REQUIRE(scratch && (reinterpret_cast<uintptr_t>(scratch) % 256) == 0, "ball_group_scratch_init: 256-byte aligned scratch");
  BxScratch sc(scratch, B);
  USIP_REQUIRE(scratch_bytes >= (int64_t)sc.total, "ball_group_scratch_init: scratch too small");
  cudaError_t e = cudaMemsetAsync(scratch, 0, sc.zero_bytes, (cudaStream_t)stream);
  if (e != cudaSuccess) { set_last_error("ball_group_scratch_init: memset"); return (int)e; }
  return 0;
}

namespace usip {
int ball_group_brute(const float* xyz, const float* feat, const float* centers, float t_max, int32_t* out_idx, float* out_group,
                     float* out_rows, int ld_rows, int B, int S, int N, int M, int K, cudaStream_t st);   // ballquery.cu
}

extern "C" int usip_ball_group_f32(const float* xyz, const float* feat, const float* centers, float radius,
                                   int32_t* out_idx, float* out_group, float* out_rows, int ld_rows, void* scratch,
                                   int64_t scratch_bytes, int B, int S, int N, int M, int K, void* stream) {
  USIP_REQUIRE(xyz && centers && out_idx && (S == 0 || feat) && B > 0 && N > 0 && M > 0 && K > 0,
               "ball_group: bad args");
  USIP_REQUIRE(!out_rows || ld_rows >= 3 + S, "ball_group: ld_rows too small");
  cudaStream_t st = (cudaStream_t)stream;
  const float t_max = radius_to_tmax_host(radius);
  const bool grid_ok = scratch && S <= 4 && (reinterpret_cast<uintptr_t>(scratch) % 256) == 0 &&
                       scratch_bytes >= usip_ball_group_scratch_bytes(B, S, N, M, K) - 256 &&
                       (!out_rows || (reinterpret_cast<uintptr_t>(out_rows) % 16) == 0);
  if (!grid_ok) return ball_group_brute(xyz, feat, centers, t_max, out_idx, out_group, out_rows, ld_rows, B, S, N, M, K, st);
  BxScratch sc(scratch, B);
  // two launches chained by programmatic dependent launch: the query grid is scheduled while the build grid drains and
  // issues its centre loads; griddepcontrol.wait orders the data.  (A third, one-CTA-per-cloud launch that publishes the
  // grid once -- instead of every build CTA deriving it -- was measured slower: 5 + 10 + 27 us against 12 + 22 us.)
  static const bool no_pdl = getenv("USIP_BALL_NO_PDL") != nullptr;            // debug aid: plain stream order instead
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization; at[0].val.programmaticStreamSerializationAllowed = 1;
  bx_build_kernel<<<dim3(cdiv(N, BX_CHUNK), B), 256, 0, st>>>(xyz, feat, centers, radius, sc.grids, sc.counts, sc.ovf_cnt,
                                                              sc.buckets, sc.ovf, S, N, M);
  int e = check_launch("bx_build_kernel");
  if (e) return e;
  const BxGrid* grids = sc.grids; const float4* bk = sc.buckets; const float4* ov = sc.ovf;
  cudaLaunchConfig_t cfg = {};
  cfg.blockDim = dim3(256); cfg.dynamicSmemBytes = 0; cfg.stream = st;
  cfg.attrs = at; cfg.numAttrs = no_pdl ? 0 : 1;
  cudaError_t ce;
  const int cpc = cdiv(M, 8);
  cfg.gridDim = dim3((unsigned)cpc, (unsigned)B);
  CUtensorMap tmap;
  int te = bx_tensor_map(&tmap, sc.buckets, B);
  if (te) return te;
  ce = cudaLaunchKernelEx(&cfg, bx_query_kernel, tmap, xyz, feat, centers, grids, sc.counts, sc.ovf_cnt, sc.done, bk, ov, t_max,
                          out_idx, out_group, out_rows, ld_rows, B, S, N, M, K, cpc);
  if (ce != cudaSuccess) { set_last_error("bx_query_kernel"); return (int)ce; }
  return check_launch("bx_query_kernel");
}
