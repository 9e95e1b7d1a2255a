// group.cu -- grouping front-end of the USIP detector (nearest-node assignment, stable cluster sort,
// cluster mean + decentring, segmented max, node kNN) and the stand-alone index_max operator.
// Reference semantics: util/som.py:17-54, models/networks.py:85-133, models/layers.py:417-421,
// models/index_max_ext/index_max_cuda.cu:9-61.
#include "common.cuh"

namespace usip {

// ------------------------------------------------------------------------------------------------
// som_assign: brute-force nearest node, node tile broadcast from shared memory, PTS points / thread.
// ------------------------------------------------------------------------------------------------
// 128 threads x 2 points: at the KITTI shape (16 clouds x 16384 points) that is 1024 CTAs, ~6.9 per SM -- 256 CTAs of
// 1024 points left 40 SMs with twice the work of the rest.
constexpr int ASSIGN_THREADS = 128;
constexpr int ASSIGN_PTS = 2;
constexpr int ASSIGN_NODE_CHUNK = 1024;  // float4 per node -> 16 KB

__global__ void __launch_bounds__(ASSIGN_THREADS)
som_assign_kernel(const float* __restrict__ xyz, const float* __restrict__ node,
                  int32_t* __restrict__ min_idx, int32_t* __restrict__ count, int N, int M) {
  __shared__ float4 snode[ASSIGN_NODE_CHUNK];
  const int b = blockIdx.y;
  const float* px = xyz + (size_t)b * 3 * N;
  const float* nx = node + (size_t)b * 3 * M;
  const int n0 = blockIdx.x * (ASSIGN_THREADS * ASSIGN_PTS) + threadIdx.x;

  float x[ASSIGN_PTS], y[ASSIGN_PTS], z[ASSIGN_PTS], best[ASSIGN_PTS];
  int bi[ASSIGN_PTS];
#pragma unroll
  for (int j = 0; j < ASSIGN_PTS; ++j) {
    int n = n0 + j * ASSIGN_THREADS;
    bool ok = n < N;
    x[j] = ok ? px[n] : 0.f; y[j] = ok ? px[N + n] : 0.f; z[j] = ok ? px[2 * N + n] : 0.f;
    best[j] = INFINITY; bi[j] = 0;
  }
  for (int m0 = 0; m0 < M; m0 += ASSIGN_NODE_CHUNK) {
    int mc = min(ASSIGN_NODE_CHUNK, M - m0);
    __syncthreads();
    for (int i = threadIdx.x; i < mc; i += ASSIGN_THREADS)
      snode[i] = make_float4(nx[m0 + i], nx[M + m0 + i], nx[2 * M + m0 + i], 0.f);
    __syncthreads();
#pragma unroll 4
    for (int m = 0; m < mc; ++m) {
      float4 nd = snode[m];
#pragma unroll
      for (int j = 0; j < ASSIGN_PTS; ++j) {
        float d = sqdist_rn(x[j], y[j], z[j], nd.x, nd.y, nd.z);
        if (d < best[j]) { best[j] = d; bi[j] = m0 + m; }
      }
    }
  }
#pragma unroll
  for (int j = 0; j < ASSIGN_PTS; ++j) {
    int n = n0 + j * ASSIGN_THREADS;
    if (n < N) {
      min_idx[(size_t)b * N + n] = bi[j];
      if (count) atomicAdd(&count[(size_t)b * M + bi[j]], 1);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Stable counting sort by node id: chunk histograms -> per-cloud scan -> placement.
// ------------------------------------------------------------------------------------------------
constexpr int SORT_CHUNK = 256;

__device__ __forceinline__ void chunk_rank(const int* keys, int tid, int key, int& rank, bool& later) {
  rank = 0; later = false;
  for (int j = 0; j < SORT_CHUNK; ++j) {
    int kj = keys[j];
    bool same = (kj == key);
    rank += (same && j < tid) ? 1 : 0;
    later = later || (same && j > tid);
  }
}

__global__ void __launch_bounds__(SORT_CHUNK)
sort_hist_kernel(const int32_t* __restrict__ min_idx, int32_t* __restrict__ hist, int N, int M, int chunks) {
  __shared__ int keys[SORT_CHUNK];
  const int b = blockIdx.y, chunk = blockIdx.x, tid = threadIdx.x;
  const int n = chunk * SORT_CHUNK + tid;
  const int key = n < N ? min_idx[(size_t)b * N + n] : -1 - tid;  // unique negatives never match
  keys[tid] = key;
  int32_t* h = hist + ((size_t)b * chunks + chunk) * M;
  for (int m = tid; m < M; m += SORT_CHUNK) h[m] = 0;
  __syncthreads();
  int rank; bool later;
  chunk_rank(keys, tid, key, rank, later);
  if (key >= 0 && !later) h[key] = rank + 1;
}

// Warp-match variants (M <= 4096): per-warp key counts in shared memory instead of the O(chunk^2) rank loop.
__global__ void __launch_bounds__(SORT_CHUNK)
sort_hist_match_kernel(const int32_t* __restrict__ min_idx, int32_t* __restrict__ hist, int N, int M, int chunks) {
  extern __shared__ unsigned short cnt[];               // [8][M]
  const int b = blockIdx.y, chunk = blockIdx.x, tid = threadIdx.x, w = tid >> 5, lane = tid & 31;
  for (int i = tid; i < 8 * M; i += SORT_CHUNK) cnt[i] = 0;
  __syncthreads();
  const int n = chunk * SORT_CHUNK + tid;
  const int key = n < N ? min_idx[(size_t)b * N + n] : -1 - tid;
  const unsigned m = __match_any_sync(0xffffffffu, key);
  if (key >= 0 && (m & ((1u << lane) - 1u)) == 0) cnt[w * M + key] = (unsigned short)__popc(m);
  __syncthreads();
  int32_t* h = hist + ((size_t)b * chunks + chunk) * M;
  for (int mm = tid; mm < M; mm += SORT_CHUNK) {
    int s = 0;
#pragma unroll
    for (int ww = 0; ww < 8; ++ww) s += cnt[ww * M + mm];
    h[mm] = s;
  }
}

__global__ void __launch_bounds__(SORT_CHUNK)
sort_place_match_kernel(const int32_t* __restrict__ min_idx, const int32_t* __restrict__ hist,
                        const int32_t* __restrict__ seg_off, int32_t* __restrict__ perm,
                        int32_t* __restrict__ row_seg, int N, int M, int chunks) {
  extern __shared__ unsigned short cnt[];               // [8][M]
  const int b = blockIdx.y, chunk = blockIdx.x, tid = threadIdx.x, w = tid >> 5, lane = tid & 31;
  for (int i = tid; i < 8 * M; i += SORT_CHUNK) cnt[i] = 0;
  __syncthreads();
  const int n = chunk * SORT_CHUNK + tid;
  const int key = n < N ? min_idx[(size_t)b * N + n] : -1 - tid;
  const unsigned m = __match_any_sync(0xffffffffu, key);
  const int below = __popc(m & ((1u << lane) - 1u));
  if (key >= 0 && below == 0) cnt[w * M + key] = (unsigned short)__popc(m);
  __syncthreads();
  if (key >= 0) {
    int rank = below;
    for (int ww = 0; ww < w; ++ww) rank += cnt[ww * M + key];
    const int pos = seg_off[(size_t)b * (M + 1) + key] + hist[((size_t)b * chunks + chunk) * M + key] + rank;
    perm[(size_t)b * N + pos] = n;
    row_seg[(size_t)b * N + pos] = b * M + key;
  }
}

__global__ void __launch_bounds__(1024)
sort_scan_kernel(int32_t* __restrict__ hist, int32_t* __restrict__ seg_off, int N, int M, int chunks) {
  extern __shared__ int tot[];          // M totals, then 1024 partials
  int* part = tot + M;
  const int b = blockIdx.x, tid = threadIdx.x, nt = blockDim.x;
  for (int m = tid; m < M; m += nt) {
    int run = 0;
    int32_t* base = hist + (size_t)b * chunks * M + m;
    int c = 0;
    for (; c + 16 <= chunks; c += 16) {          // 16 independent loads in flight, then the serial prefix
      int h[16];
#pragma unroll
      for (int u = 0; u < 16; ++u) h[u] = base[(size_t)(c + u) * M];
#pragma unroll
      for (int u = 0; u < 16; ++u) { base[(size_t)(c + u) * M] = run; run += h[u]; }
    }
    for (; c < chunks; ++c) { int h = base[(size_t)c * M]; base[(size_t)c * M] = run; run += h; }
    tot[m] = run;
  }
  __syncthreads();
  // exclusive scan of tot[0..M): each thread owns a contiguous slice
  const int per = (M + nt - 1) / nt;
  const int lo = min(tid * per, M), hi = min(lo + per, M);
  int s = 0;
  for (int m = lo; m < hi; ++m) s += tot[m];
  // block-wide exclusive scan of the per-thread sums by warp shuffles (a serial pass of thread 0 over the 1024 partials
  // was most of this kernel's 13 us)
  const int lane = tid & 31, warp = tid >> 5;
  int inc = s;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const int v = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += v; }
  if (lane == 31) part[warp] = inc;
  __syncthreads();
  if (warp == 0) {
    int v = lane < (nt >> 5) ? part[lane] : 0;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const int u = __shfl_up_sync(0xffffffffu, v, o); if (lane >= o) v += u; }
    part[lane] = v;
  }
  __syncthreads();
  int run = inc - s + (warp > 0 ? part[warp - 1] : 0);
  for (int m = lo; m < hi; ++m) { seg_off[(size_t)b * (M + 1) + m] = run; run += tot[m]; }
  if (tid == 0) seg_off[(size_t)b * (M + 1) + M] = N;
}

__global__ void __launch_bounds__(SORT_CHUNK)
sort_place_kernel(const int32_t* __restrict__ min_idx, const int32_t* __restrict__ hist,
                  const int32_t* __restrict__ seg_off, int32_t* __restrict__ perm,
                  int32_t* __restrict__ row_seg, int N, int M, int chunks) {
  __shared__ int keys[SORT_CHUNK];
  const int b = blockIdx.y, chunk = blockIdx.x, tid = threadIdx.x;
  const int n = chunk * SORT_CHUNK + tid;
  const int key = n < N ? min_idx[(size_t)b * N + n] : -1 - tid;
  keys[tid] = key;
  __syncthreads();
  int rank; bool later;
  chunk_rank(keys, tid, key, rank, later);
  if (key >= 0) {
    int pos = seg_off[(size_t)b * (M + 1) + key] + hist[((size_t)b * chunks + chunk) * M + key] + rank;
    perm[(size_t)b * N + pos] = n;
    row_seg[(size_t)b * N + pos] = b * M + key;
  }
}

// ------------------------------------------------------------------------------------------------
// cluster mean + decentre + concat: one warp per (cloud, node).
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
cluster_mean_decenter_kernel(const float* __restrict__ xyz, const float* __restrict__ feat,
                             const int32_t* __restrict__ seg_off, const int32_t* __restrict__ perm,
                             float* __restrict__ cluster_mean, float* __restrict__ x_aug, int ldx,
                             int B, int S, int N, int M) {
  const int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (w >= B * M) return;
  const int b = w / M, m = w - b * M;
  const int s = seg_off[(size_t)b * (M + 1) + m], e = seg_off[(size_t)b * (M + 1) + m + 1];
  const float* px = xyz + (size_t)b * 3 * N;
  const int32_t* pp = perm + (size_t)b * N;
  float sx = 0.f, sy = 0.f, sz = 0.f;
  for (int r = s + lane; r < e; r += 32) {
    int n = pp[r];
    sx += px[n]; sy += px[N + n]; sz += px[2 * N + n];
  }
  sx = warp_sum(sx); sy = warp_sum(sy); sz = warp_sum(sz);
  const float den = (float)(e - s) + 1e-5f;               // networks.py:96-97
  const float mx = sx / den, my = sy / den, mz = sz / den;
  if (lane == 0) {
    cluster_mean[(size_t)b * 3 * M + m] = mx;
    cluster_mean[(size_t)b * 3 * M + M + m] = my;
    cluster_mean[(size_t)b * 3 * M + 2 * M + m] = mz;
  }
  const float* pf = feat ? feat + (size_t)b * S * N : nullptr;
  if (ldx == 8 && S <= 5 && (reinterpret_cast<uintptr_t>(x_aug) & 15) == 0) {
    // the usual row (xyz + <= 5 features, padded to 8 floats): two 16-byte stores per row instead of eight 4-byte ones
    for (int r = s + lane; r < e; r += 32) {
      const int n = pp[r];
      float v[8];
      v[0] = px[n] - mx; v[1] = px[N + n] - my; v[2] = px[2 * N + n] - mz;   // networks.py:105-107
#pragma unroll
      for (int c = 0; c < 5; ++c) v[3 + c] = c < S ? pf[(size_t)c * N + n] : 0.f;
      float4* o = reinterpret_cast<float4*>(x_aug + ((size_t)b * N + r) * 8);
      o[0] = make_float4(v[0], v[1], v[2], v[3]); o[1] = make_float4(v[4], v[5], v[6], v[7]);
    }
    return;
  }
  for (int r = s + lane; r < e; r += 32) {
    int n = pp[r];
    float* o = x_aug + ((size_t)b * N + r) * ldx;
    o[0] = px[n] - mx; o[1] = px[N + n] - my; o[2] = px[2 * N + n] - mz;   // networks.py:105-107
    for (int c = 0; c < S; ++c) o[3 + c] = pf[(size_t)c * N + n];
    for (int c = 3 + S; c < ldx; ++c) o[c] = 0.f;
  }
}

// ------------------------------------------------------------------------------------------------
// segmented max over the (contiguous, sorted) rows of each node; float4 channel groups per lane.
// Reference: index_max + gather (*mask_row_max) at networks.py:117-120,130-133; the `> -1000`
// floor of index_max_cuda.cu:38-49 is honoured: no winner -> the reference gathers point n=0.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
segmax_kernel(const float* __restrict__ X, int ldx, const int32_t* __restrict__ seg_off,
              const int32_t* __restrict__ perm, float* __restrict__ pooled, int ldp,
              int32_t* __restrict__ arg, int B, int N, int M, int C) {
  const int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (w >= B * M) return;
  const int b = w / M, m = w - b * M;
  const int s = seg_off[(size_t)b * (M + 1) + m], e = seg_off[(size_t)b * (M + 1) + m + 1];
  const size_t row0 = (size_t)b * N;
  auto scan = [&](int c4, int first, int step, float4& best, int4& bi) {
    for (int r = first; r < e; r += step) {
      float4 v = *reinterpret_cast<const float4*>(X + (row0 + r) * ldx + c4 * 4);
      if (v.x > best.x) { best.x = v.x; bi.x = r; }
      if (v.y > best.y) { best.y = v.y; bi.y = r; }
      if (v.z > best.z) { best.z = v.z; bi.z = r; }
      if (v.w > best.w) { best.w = v.w; bi.w = r; }
    }
  };
  auto finish = [&](int c4, float4 best, int4 bi) {
    float4 out = make_float4(0.f, 0.f, 0.f, 0.f);
    int4 oa = make_int4(-1, -1, -1, -1);
    if (e > s) {
      // no element above the -1000 floor: reference index is 0 -> value of original point n = 0
      if (bi.x < 0 || bi.y < 0 || bi.z < 0 || bi.w < 0) {
        int r0 = 0;
        for (int r = 0; r < N; ++r) if (perm[row0 + r] == 0) { r0 = r; break; }
        float4 v0 = *reinterpret_cast<const float4*>(X + (row0 + r0) * ldx + c4 * 4);
        if (bi.x < 0) { best.x = v0.x; bi.x = r0; }
        if (bi.y < 0) { best.y = v0.y; bi.y = r0; }
        if (bi.z < 0) { best.z = v0.z; bi.z = r0; }
        if (bi.w < 0) { best.w = v0.w; bi.w = r0; }
      }
      out = best;
      oa = make_int4((int)row0 + bi.x, (int)row0 + bi.y, (int)row0 + bi.z, (int)row0 + bi.w);
    }
    *reinterpret_cast<float4*>(pooled + (size_t)w * ldp + c4 * 4) = out;
    if (arg) *reinterpret_cast<int4*>(arg + (size_t)w * C + c4 * 4) = oa;
  };
  if (C <= 64) {
    // the <= 16 float4 groups of a row occupy half a warp: the two halves take alternating rows and merge at the end
    // (larger value, then smaller row = the first maximum, as the single ascending scan gives it)
    const int c4 = lane & 15, sub = lane >> 4;
    const bool active = c4 * 4 < C;
    float4 best = make_float4(-1000.f, -1000.f, -1000.f, -1000.f);
    int4 bi = make_int4(-1, -1, -1, -1);
    if (active) scan(c4, s + sub, 2, best, bi);
    const float4 ob = make_float4(__shfl_xor_sync(0xffffffffu, best.x, 16), __shfl_xor_sync(0xffffffffu, best.y, 16),
                                  __shfl_xor_sync(0xffffffffu, best.z, 16), __shfl_xor_sync(0xffffffffu, best.w, 16));
    const int4 oi = make_int4(__shfl_xor_sync(0xffffffffu, bi.x, 16), __shfl_xor_sync(0xffffffffu, bi.y, 16),
                              __shfl_xor_sync(0xffffffffu, bi.z, 16), __shfl_xor_sync(0xffffffffu, bi.w, 16));
    // an index < 0 means "nothing above the floor" on that side; a real row always beats it
    if (oi.x >= 0 && (bi.x < 0 || ob.x > best.x || (ob.x == best.x && oi.x < bi.x))) { best.x = ob.x; bi.x = oi.x; }
    if (oi.y >= 0 && (bi.y < 0 || ob.y > best.y || (ob.y == best.y && oi.y < bi.y))) { best.y = ob.y; bi.y = oi.y; }
    if (oi.z >= 0 && (bi.z < 0 || ob.z > best.z || (ob.z == best.z && oi.z < bi.z))) { best.z = ob.z; bi.z = oi.z; }
    if (oi.w >= 0 && (bi.w < 0 || ob.w > best.w || (ob.w == best.w && oi.w < bi.w))) { best.w = ob.w; bi.w = oi.w; }
    if (active && sub == 0) finish(c4, best, bi);
    return;
  }
  for (int c4 = lane; c4 * 4 < C; c4 += 32) {
    float4 best = make_float4(-1000.f, -1000.f, -1000.f, -1000.f);
    int4 bi = make_int4(-1, -1, -1, -1);
    scan(c4, s, 1, best, bi);
    finish(c4, best, bi);
  }
}

// ------------------------------------------------------------------------------------------------
// node kNN: one warp per query node, distances in shared memory, K rounds of warp arg-min on the
// packed key (sqrt-distance bits << 32 | index): ascending distance, ties by ascending index.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
knn_nodes_kernel(const float* __restrict__ pts, int32_t* __restrict__ knn_idx, int B, int M, int K) {
  extern __shared__ unsigned long long skey[];     // 8 warps x M packed keys (distance bits << 32 | index), built once
  const int wib = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int w = blockIdx.x * 8 + wib;
  if (w >= B * M) return;
  const int b = w / M, m = w - b * M;
  const float* p = pts + (size_t)b * 3 * M;
  unsigned long long* d = skey + (size_t)wib * M;
  const float qx = p[m], qy = p[M + m], qz = p[2 * M + m];
  for (int j = lane; j < M; j += 32)
    d[j] = ((unsigned long long)__float_as_uint(__fsqrt_rn(sqdist_rn(qx, qy, qz, p[j], p[M + j], p[2 * M + j]))) << 32) | (unsigned)j;
  __syncwarp();
  for (int k = 0; k < K; ++k) {
    unsigned long long best = ~0ull;
    for (int j = lane; j < M; j += 32) { const unsigned long long key = d[j]; best = key < best ? key : best; }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const unsigned long long other = __shfl_xor_sync(0xffffffffu, best, o);
      best = other < best ? other : best;
    }
    int j = (int)(best & 0xffffffffu);
    if (k >= M) j = 0;                             // K > M: undefined in the reference (topk would throw)
    if (lane == 0) knn_idx[(size_t)w * K + k] = j;
    if (lane == (j & 31) && k < M) d[j] = ~0ull;   // taken: the largest key
    __syncwarp();
  }
}

// Register variant for M <= 32*KPL nodes: lane l keeps the fp32 distance bits of nodes l, l+32, ... in registers (the node
// index is implied by the slot), so a selection round is 16 register compares + one (distance, index) warp reduction instead
// of 16 eight-byte shared-memory loads per lane (the shared-memory kernel above spends its time in that traffic: 512
// wavefronts per query).  Same order as the packed key: ascending sqrt-distance bits, ties by ascending node index.
template <int KPL>
__global__ void __launch_bounds__(256)
knn_nodes_reg_kernel(const float* __restrict__ pts, int32_t* __restrict__ knn_idx, int B, int M, int K) {
  const int wib = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int w = blockIdx.x * 8 + wib;
  if (w >= B * M) return;
  const int b = w / M, m = w - b * M;
  const float* p = pts + (size_t)b * 3 * M;
  const float qx = __ldg(p + m), qy = __ldg(p + M + m), qz = __ldg(p + 2 * M + m);
  uint32_t d[KPL];
#pragma unroll
  for (int i = 0; i < KPL; ++i) {
    const int j = lane + 32 * i;
    d[i] = j < M ? __float_as_uint(__fsqrt_rn(sqdist_rn(qx, qy, qz, __ldg(p + j), __ldg(p + M + j), __ldg(p + 2 * M + j)))) : 0xffffffffu;
  }
  for (int k = 0; k < K; ++k) {
    uint32_t bd = d[0]; int bi = 0;
#pragma unroll
    for (int i = 1; i < KPL; ++i) if (d[i] < bd) { bd = d[i]; bi = i; }   // strict: the smallest slot (= index) on ties
    int bj = lane + 32 * bi;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const uint32_t od = __shfl_xor_sync(0xffffffffu, bd, o); const int oj = __shfl_xor_sync(0xffffffffu, bj, o);
      if (od < bd || (od == bd && oj < bj)) { bd = od; bj = oj; }
    }
    int j = bj;
    if (k >= M) j = 0;                             // K > M: undefined in the reference (topk would throw)
    if (lane == 0) knn_idx[(size_t)w * K + k] = j;
    if (lane == (bj & 31) && k < M) {
      const int slot = bj >> 5;
#pragma unroll
      for (int i = 0; i < KPL; ++i) if (i == slot) d[i] = 0xffffffffu;   // taken (a padded slot can never win again either)
    }
  }
}

// ------------------------------------------------------------------------------------------------
// stand-alone index_max (reference operator).  CTA = (cloud, CPB channels); running maxima live in
// shared memory as packed u64 (ordered value << 32 | ~n) with a 32-bit filter word read first, so
// only ~H(cluster size) elements per cluster take the 64-bit atomicMax path.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ unsigned long long im_init_key() {
  return ((unsigned long long)f2ord(-1000.0f) << 32) | 0xffffffffull;
}

template <int CPB>
__global__ void __launch_bounds__(256)
index_max_smem_kernel(const float* __restrict__ data, const int32_t* __restrict__ index,
                      int32_t* __restrict__ out_idx, int C, int N, int K) {
  extern __shared__ unsigned long long skey[];     // CPB*K packed keys, then CPB*K u32 filters
  uint32_t* sfil = reinterpret_cast<uint32_t*>(skey + (size_t)CPB * K);
  const int b = blockIdx.y, c0 = blockIdx.x * CPB;
  const int tid = threadIdx.x;
  const unsigned long long init = im_init_key();
  for (int i = tid; i < CPB * K; i += 256) { skey[i] = init; sfil[i] = (uint32_t)(init >> 32); }
  __syncthreads();
  const int32_t* idx = index + (size_t)b * N;
  const float* base = data + ((size_t)b * C + c0) * N;
  const int nch = min(CPB, C - c0);
  // int4 / float4 loads need every row start 16-byte aligned: N % 4 == 0 keeps the rows in step with the base pointers,
  // which a view at an element offset (e.g. buf[1:]) does not align
  const bool vec_ok = (N % 4 == 0) && ((reinterpret_cast<uintptr_t>(data) | reinterpret_cast<uintptr_t>(index)) & 15) == 0;
  if (vec_ok) {
    for (int n4 = tid; n4 * 4 < N; n4 += 256) {
      int4 k4 = *reinterpret_cast<const int4*>(idx + n4 * 4);
      float4 v[CPB];
#pragma unroll
      for (int c = 0; c < CPB; ++c)
        v[c] = c < nch ? *reinterpret_cast<const float4*>(base + (size_t)c * N + n4 * 4) : make_float4(0, 0, 0, 0);
#pragma unroll
      for (int c = 0; c < CPB; ++c) {
        if (c >= nch) break;
        const float vv[4] = {v[c].x, v[c].y, v[c].z, v[c].w};
        const int kk[4] = {k4.x, k4.y, k4.z, k4.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          float val = __fadd_rn(vv[j], 0.0f);                     // -0 -> +0 ('>' treats them equal)
          if (val != val) continue;                               // NaN never wins a '>' test
          uint32_t o = f2ord(val);
          int slot = c * K + kk[j];
          if (o >= sfil[slot]) {
            unsigned long long key = ((unsigned long long)o << 32) | (uint32_t)(~(uint32_t)(n4 * 4 + j));
            unsigned long long old = atomicMax(&skey[slot], key);
            if (key > old) atomicMax(&sfil[slot], o);
          }
        }
      }
    }
  } else {
    for (int n = tid; n < N; n += 256) {
      int k = idx[n];
      for (int c = 0; c < nch; ++c) {
        float val = __fadd_rn(base[(size_t)c * N + n], 0.0f);
        if (val != val) continue;
        uint32_t o = f2ord(val);
        int slot = c * K + k;
        if (o >= sfil[slot]) {
          unsigned long long key = ((unsigned long long)o << 32) | (uint32_t)(~(uint32_t)n);
          unsigned long long old = atomicMax(&skey[slot], key);
          if (key > old) atomicMax(&sfil[slot], o);
        }
      }
    }
  }
  __syncthreads();
  for (int i = tid; i < nch * K; i += 256) {
    int c = i / K, k = i - c * K;
    out_idx[((size_t)b * C + c0 + c) * K + k] = (int32_t)(~(uint32_t)(skey[i] & 0xffffffffull));
  }
}

// global-memory variant for very large K (no shared-memory cap at all)
__global__ void index_max_init_kernel(unsigned long long* scratch, size_t n) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) scratch[i] = im_init_key();
}
__global__ void __launch_bounds__(256)
index_max_global_kernel(const float* __restrict__ data, const int32_t* __restrict__ index,
                        unsigned long long* __restrict__ scratch, int C, int N, int K) {
  const int b = blockIdx.z, c = blockIdx.y;
  const int n = blockIdx.x * 256 + threadIdx.x;
  if (n >= N) return;
  float val = __fadd_rn(data[((size_t)b * C + c) * N + n], 0.0f);
  if (val != val) return;
  int k = index[(size_t)b * N + n];
  unsigned long long key = ((unsigned long long)f2ord(val) << 32) | (uint32_t)(~(uint32_t)n);
  unsigned long long* p = scratch + ((size_t)b * C + c) * K + k;
  if (key > *p) atomicMax(p, key);
}
__global__ void index_max_decode_kernel(const unsigned long long* scratch, int32_t* out, size_t n) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = (int32_t)(~(uint32_t)(scratch[i] & 0xffffffffull));
}

// knn_gather_by_indexing (operations.py:271-287)
__global__ void knn_gather_kernel(const float* __restrict__ src, const int32_t* __restrict__ idx,
                                  float* __restrict__ out, int C, int N, int MK, size_t total) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  int mk = (int)(i % MK); size_t bc = i / MK; int b = (int)(bc / C);
  out[i] = src[bc * N + idx[(size_t)b * MK + mk]];
}

template <int CPB>
static int launch_index_max_smem(const float* data, const int32_t* index, int32_t* out, int B, int C, int N, int K,
                                 cudaStream_t st) {
  size_t smem = (size_t)CPB * K * 12;
  cudaError_t e = cudaFuncSetAttribute(index_max_smem_kernel<CPB>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) { set_last_error("index_max smem attr"); return (int)e; }
  dim3 grid(cdiv(C, CPB), B);
  index_max_smem_kernel<CPB><<<grid, 256, smem, st>>>(data, index, out, C, N, K);
  return check_launch("index_max_smem_kernel");
}

bool index_max_bucket_ok(const float* data, int N, int K);                                    // indexmax.cu
int launch_index_max_bucket(const float* data, const int32_t* index, int32_t* out, int B, int C, int N, int K, cudaStream_t st);

}  // namespace usip

using namespace usip;

extern "C" int usip_index_max_f32(const float* data, const int32_t* index, int32_t* out_idx,
                                  unsigned long long* scratch, int B, int C, int N, int K, void* stream) {
  USIP_REQUIRE(data && index && out_idx && B > 0 && C > 0 && N > 0 && K > 0, "index_max: bad args");
  cudaStream_t st = (cudaStream_t)stream;
  // enough rows per cloud to amortise the per-cloud bucket sort: the HBM-speed kernel; else the atomic-max kernels below
  if (C >= 8 && (long long)B * C >= 64 && index_max_bucket_ok(data, N, K)) return launch_index_max_bucket(data, index, out_idx, B, C, N, K, st);
  const size_t budget = 96 * 1024;   // keep >= 2 CTAs / SM
  if ((size_t)8 * K * 12 <= budget && C >= 8) return launch_index_max_smem<8>(data, index, out_idx, B, C, N, K, st);
  if ((size_t)4 * K * 12 <= budget && C >= 4) return launch_index_max_smem<4>(data, index, out_idx, B, C, N, K, st);
  if ((size_t)2 * K * 12 <= budget && C >= 2) return launch_index_max_smem<2>(data, index, out_idx, B, C, N, K, st);
  if ((size_t)1 * K * 12 <= 200 * 1024) return launch_index_max_smem<1>(data, index, out_idx, B, C, N, K, st);
  USIP_REQUIRE(scratch, "index_max: scratch required for very large K");
  size_t tot = (size_t)B * C * K;
  index_max_init_kernel<<<(unsigned)cdiv64(tot, 256), 256, 0, st>>>(scratch, tot);
  dim3 grid(cdiv(N, 256), C, B);
  index_max_global_kernel<<<grid, 256, 0, st>>>(data, index, scratch, C, N, K);
  index_max_decode_kernel<<<(unsigned)cdiv64(tot, 256), 256, 0, st>>>(scratch, out_idx, tot);
  return check_launch("index_max_global");
}

extern "C" int usip_knn_gather_f32(const float* src, const int32_t* idx, float* out,
                                   int B, int C, int N, int M, int K, void* stream) {
  USIP_REQUIRE(src && idx && out, "knn_gather: bad args");
  size_t total = (size_t)B * C * M * K;
  knn_gather_kernel<<<(unsigned)cdiv64(total, 256), 256, 0, (cudaStream_t)stream>>>(src, idx, out, C, N, M * K, total);
  return check_launch("knn_gather_kernel");
}

extern "C" int usip_som_assign_f32(const float* xyz, const float* node, int32_t* min_idx, int32_t* count,
                                   int B, int N, int M, void* stream) {
  USIP_REQUIRE(xyz && node && min_idx && B > 0 && N > 0 && M > 0, "som_assign: bad args");
  dim3 grid(cdiv(N, ASSIGN_THREADS * ASSIGN_PTS), B);
  som_assign_kernel<<<grid, ASSIGN_THREADS, 0, (cudaStream_t)stream>>>(xyz, node, min_idx, count, N, M);
  return check_launch("som_assign_kernel");
}

extern "C" int usip_cluster_sort(const int32_t* min_idx, int32_t* seg_off, int32_t* perm, int32_t* row_seg,
                                 int32_t* scratch, int B, int N, int M, void* stream) {
  USIP_REQUIRE(min_idx && seg_off && perm && row_seg && scratch, "cluster_sort: bad args");
  cudaStream_t st = (cudaStream_t)stream;
  const int chunks = cdiv(N, SORT_CHUNK);
  dim3 grid(chunks, B);
  const bool match = M <= 4096;
  const size_t msm = (size_t)8 * M * sizeof(unsigned short);
  if (match) {
    if (msm > 48 * 1024) {
      cudaFuncSetAttribute(sort_hist_match_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)msm);
      cudaFuncSetAttribute(sort_place_match_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)msm);
    }
    sort_hist_match_kernel<<<grid, SORT_CHUNK, msm, st>>>(min_idx, scratch, N, M, chunks);
  } else {
    sort_hist_kernel<<<grid, SORT_CHUNK, 0, st>>>(min_idx, scratch, N, M, chunks);
  }
  size_t smem = (size_t)(M + 1024) * sizeof(int);
  USIP_REQUIRE(smem <= 200 * 1024, "cluster_sort: M too large");
  if (smem > 48 * 1024) cudaFuncSetAttribute(sort_scan_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  sort_scan_kernel<<<B, 1024, smem, st>>>(scratch, seg_off, N, M, chunks);
  if (match) sort_place_match_kernel<<<grid, SORT_CHUNK, msm, st>>>(min_idx, scratch, seg_off, perm, row_seg, N, M, chunks);
  else sort_place_kernel<<<grid, SORT_CHUNK, 0, st>>>(min_idx, scratch, seg_off, perm, row_seg, N, M, chunks);
  return check_launch("cluster_sort");
}

extern "C" int usip_cluster_mean_decenter(const float* xyz, const float* feat, const int32_t* seg_off,
                                          const int32_t* perm, float* cluster_mean, float* x_aug, int ldx,
                                          int B, int S, int N, int M, void* stream) {
  USIP_REQUIRE(xyz && seg_off && perm && cluster_mean && x_aug && ldx >= 3 + S && (S == 0 || feat),
               "cluster_mean_decenter: bad args");
  int warps = B * M;
  cluster_mean_decenter_kernel<<<cdiv(warps * 32, 256), 256, 0, (cudaStream_t)stream>>>(
      xyz, feat, seg_off, perm, cluster_mean, x_aug, ldx, B, S, N, M);
  return check_launch("cluster_mean_decenter_kernel");
}

extern "C" int usip_segmax(const float* X, int ldx, const int32_t* seg_off, const int32_t* perm,
                           float* pooled, int ldp, int32_t* arg, int B, int N, int M, int C, void* stream) {
  USIP_REQUIRE(X && seg_off && perm && pooled && C % 4 == 0 && ldx % 4 == 0 && ldp % 4 == 0, "segmax: bad args");
  // the kernel reads X and writes pooled as float4, arg as int4
  USIP_REQUIRE(((reinterpret_cast<uintptr_t>(X) | reinterpret_cast<uintptr_t>(pooled) | reinterpret_cast<uintptr_t>(arg)) & 15) == 0,
               "segmax: X, pooled and arg must be 16-byte aligned");
  int warps = B * M;
  segmax_kernel<<<cdiv(warps * 32, 256), 256, 0, (cudaStream_t)stream>>>(X, ldx, seg_off, perm, pooled, ldp, arg,
                                                                       B, N, M, C);
  return check_launch("segmax_kernel");
}

extern "C" int usip_knn_nodes(const float* pts, int32_t* knn_idx, int B, int M, int K, void* stream) {
  USIP_REQUIRE(pts && knn_idx && K > 0 && M > 0, "knn_nodes: bad args");
  if (M <= 512 && K <= M) {                       // keys in registers (16 per lane)
    knn_nodes_reg_kernel<16><<<cdiv(B * M, 8), 256, 0, (cudaStream_t)stream>>>(pts, knn_idx, B, M, K);
    return check_launch("knn_nodes_reg_kernel");
  }
  size_t smem = (size_t)8 * M * sizeof(unsigned long long);
  USIP_REQUIRE(smem <= 200 * 1024, "knn_nodes: M too large");
  if (smem > 48 * 1024) cudaFuncSetAttribute(knn_nodes_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  knn_nodes_kernel<<<cdiv(B * M, 8), 256, smem, (cudaStream_t)stream>>>(pts, knn_idx, B, M, K);
  return check_launch("knn_nodes_kernel");
}
