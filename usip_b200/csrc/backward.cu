// backward.cu -- backward pass of the fused detector / descriptor plan.
//
// Autograd of the reference graph (models/networks.py:75-162, models/layers.py) re-derived for the fused
// forward plan: train-mode BatchNorm backward is "reduce (sum g, sum g*xhat) -> finalize -> apply", the dgrad
// GEMMs reuse usip_layer_fwd with a transposed weight view, the wgrad GEMMs reduce over the row dimension
// with the same register-tiled micro-kernel as the forward SIMT path, and every gather of the forward
// (arg-max pooling, un-pooling, kNN grouping, group max) has its scatter here.
#include "common.cuh"

namespace usip {

constexpr int BW_ROWS = 128;      // rows per reduction tile (same as the forward stat tile)

// ------------------------------------------------------------------------------------------------
// BatchNorm(+ReLU) backward, phase 1: partial sums of g_z and g_z * xhat,  g_z = g * 1[scale*y+shift > 0].
// part holds cdiv(P,128) rows of [2][C]; CTA i accumulates the 128-row tiles i, i+grid, ... into row i and the rows past
// the grid are written as zeros, so the finalize kernel sums the same number of rows whatever the grid is.
// Fast kernel (C/4 divides 256): a thread owns one 4-column group, streams rows with independent loads in flight.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
bn_bwd_reduce_kernel(const float* __restrict__ G, int ldg, const float* __restrict__ Y, int ldy,
                     const float* __restrict__ scale, const float* __restrict__ shift,
                     const float* __restrict__ mean, const float* __restrict__ invstd, int relu,
                     float* __restrict__ part, int P, int C, int ntiles) {
  __shared__ float red[2][256][4];
  const int c4n = C >> 2, rpp = 256 / c4n;
  const int cgp = threadIdx.x % c4n, c = cgp * 4, rl = threadIdx.x / c4n;
  const float4 sc = *reinterpret_cast<const float4*>(scale + c), sh = *reinterpret_cast<const float4*>(shift + c);
  const float4 mu = *reinterpret_cast<const float4*>(mean + c), is = *reinterpret_cast<const float4*>(invstd + c);
  const float scv[4] = {sc.x, sc.y, sc.z, sc.w}, shv[4] = {sh.x, sh.y, sh.z, sh.w};
  const float muv[4] = {mu.x, mu.y, mu.z, mu.w}, isv[4] = {is.x, is.y, is.z, is.w};
  float s1[4] = {0, 0, 0, 0}, s2[4] = {0, 0, 0, 0};
  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int rend = min(P, (tile + 1) * BW_ROWS);
    for (int r0 = tile * BW_ROWS + rl; r0 < rend; r0 += 4 * rpp) {
      float4 g4[4], y4[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int r = r0 + u * rpp;
        if (r < rend) {
          g4[u] = __ldg(reinterpret_cast<const float4*>(G + (size_t)r * ldg + c));
          y4[u] = __ldg(reinterpret_cast<const float4*>(Y + (size_t)r * ldy + c));
        }
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        if (r0 + u * rpp < rend) {
          const float gv[4] = {g4[u].x, g4[u].y, g4[u].z, g4[u].w}, yv[4] = {y4[u].x, y4[u].y, y4[u].z, y4[u].w};
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const float z = fmaf(yv[j], scv[j], shv[j]);
            const float gz = (!relu || z > 0.f) ? gv[j] : 0.f;
            s1[j] += gz; s2[j] = fmaf(gz, (yv[j] - muv[j]) * isv[j], s2[j]);
          }
        }
      }
    }
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) { red[0][threadIdx.x][j] = s1[j]; red[1][threadIdx.x][j] = s2[j]; }
  __syncthreads();
  if (threadIdx.x < c4n) {
    float a[4] = {0, 0, 0, 0}, bsum[4] = {0, 0, 0, 0};
    for (int k = 0; k < rpp; ++k)
#pragma unroll
      for (int j = 0; j < 4; ++j) { a[j] += red[0][k * c4n + threadIdx.x][j]; bsum[j] += red[1][k * c4n + threadIdx.x][j]; }
    float* o = part + (size_t)blockIdx.x * 2 * C + threadIdx.x * 4;
    *reinterpret_cast<float4*>(o) = make_float4(a[0], a[1], a[2], a[3]);
    *reinterpret_cast<float4*>(o + C) = make_float4(bsum[0], bsum[1], bsum[2], bsum[3]);
  }
  // partial rows no CTA owns
  for (int t = gridDim.x + blockIdx.x; t < ntiles; t += gridDim.x)
    for (int i = threadIdx.x; i < 2 * C; i += 256) part[(size_t)t * 2 * C + i] = 0.f;
}

// generic variant: CTA = one 128-row tile x min(C,128) channels
__global__ void __launch_bounds__(256)
bn_bwd_reduce_tile_kernel(const float* __restrict__ G, int ldg, const float* __restrict__ Y, int ldy,
                          const float* __restrict__ scale, const float* __restrict__ shift,
                          const float* __restrict__ mean, const float* __restrict__ invstd, int relu,
                          float* __restrict__ part, int P, int C) {
  __shared__ float red[2][32][132];
  const int CW = min(C, 128), c4n = CW / 4, rsn = 256 / c4n;
  const int tile = blockIdx.x, cb = blockIdx.y * 128;
  const int c4 = threadIdx.x % c4n, rs = threadIdx.x / c4n;
  const int c = cb + c4 * 4;
  float s1[4] = {0, 0, 0, 0}, s2[4] = {0, 0, 0, 0};
  if (c < C) {
    const float4 sc = *reinterpret_cast<const float4*>(scale + c), sh = *reinterpret_cast<const float4*>(shift + c);
    const float4 mu = *reinterpret_cast<const float4*>(mean + c), is = *reinterpret_cast<const float4*>(invstd + c);
    const float scv[4] = {sc.x, sc.y, sc.z, sc.w}, shv[4] = {sh.x, sh.y, sh.z, sh.w};
    const float muv[4] = {mu.x, mu.y, mu.z, mu.w}, isv[4] = {is.x, is.y, is.z, is.w};
    const int rend = min(P, (tile + 1) * BW_ROWS);
    for (int r = tile * BW_ROWS + rs; r < rend; r += rsn) {
      const float4 g4 = *reinterpret_cast<const float4*>(G + (size_t)r * ldg + c);
      const float4 y4 = *reinterpret_cast<const float4*>(Y + (size_t)r * ldy + c);
      const float gv[4] = {g4.x, g4.y, g4.z, g4.w}, yv[4] = {y4.x, y4.y, y4.z, y4.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float z = fmaf(yv[j], scv[j], shv[j]);
        const float gz = (!relu || z > 0.f) ? gv[j] : 0.f;
        s1[j] += gz; s2[j] = fmaf(gz, (yv[j] - muv[j]) * isv[j], s2[j]);
      }
    }
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) { red[0][rs][c4 * 4 + j] = s1[j]; red[1][rs][c4 * 4 + j] = s2[j]; }
  __syncthreads();
  if (threadIdx.x < CW && cb + threadIdx.x < C) {
    float a = 0.f, b = 0.f;
    for (int t = 0; t < rsn; ++t) { a += red[0][t][threadIdx.x]; b += red[1][t][threadIdx.x]; }
    part[((size_t)tile * 2 + 0) * C + cb + threadIdx.x] = a;
    part[((size_t)tile * 2 + 1) * C + cb + threadIdx.x] = b;
  }
}

// phase 2: reduce partials (double, fixed order) -> g_gamma = sum g_z*xhat, g_beta = sum g_z, c1 = g_beta/n, c2 = g_gamma/n
__global__ void __launch_bounds__(256)
bn_bwd_finalize_kernel(const float* __restrict__ part, int ntiles, double count, int C, float* __restrict__ g_gamma,
                       float* __restrict__ g_beta, float* __restrict__ c1, float* __restrict__ c2, int accumulate) {
  // 8 channels x 32 partial-row slices per CTA (C/8 CTAs; 32 channels per CTA left a 64-channel layer with 2 CTAs and a
  // serial tail of dependent loads: 17 us); batches of 8 predicated loads, two warp shuffles, one barrier
  __shared__ double sh[2][8][8];
  const int cl = threadIdx.x & 7, sl = threadIdx.x >> 3;
  const int c = blockIdx.x * 8 + cl;
  double a = 0.0, b = 0.0;
  if (c < C) {
    for (int t = sl; t < ntiles; t += 8 * 32) {
      // sixteen loads in flight per batch: rows past the end are read from the last row (a valid address, no branch around
      // the load -- predicated loads compiled to sixteen serialised round trips, 59 us) and dropped afterwards
      float x[8], y[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const int tt = min(t + u * 32, ntiles - 1);
        x[u] = __ldg(part + ((size_t)tt * 2 + 0) * C + c);
        y[u] = __ldg(part + ((size_t)tt * 2 + 1) * C + c);
      }
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const bool ok = t + u * 32 < ntiles;
        a += ok ? (double)x[u] : 0.0; b += ok ? (double)y[u] : 0.0;
      }
    }
  }
  a += __shfl_xor_sync(0xffffffffu, a, 8); b += __shfl_xor_sync(0xffffffffu, b, 8);
  a += __shfl_xor_sync(0xffffffffu, a, 16); b += __shfl_xor_sync(0xffffffffu, b, 16);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane < 8) { sh[0][warp][lane] = a; sh[1][warp][lane] = b; }
  __syncthreads();
  if (sl == 0 && c < C) {
    double A = 0.0, B = 0.0;
#pragma unroll
    for (int t = 0; t < 8; ++t) { A += sh[0][t][cl]; B += sh[1][t][cl]; }
    if (g_beta) g_beta[c] = (accumulate ? g_beta[c] : 0.f) + (float)A;
    if (g_gamma) g_gamma[c] = (accumulate ? g_gamma[c] : 0.f) + (float)B;
    c1[c] = (float)(A / count); c2[c] = (float)(B / count);
  }
}

// phase 3: g_y = scale * (g_z - c1 - xhat*c2)            (scale = gamma*invstd)
// HBM-bound (2 reads + 1 write of [P,C]): a thread owns one 4-column group -- its six per-channel vectors live in
// registers -- and streams rows with four independent row loads in flight.  (C/4 divides 256.)
__global__ void __launch_bounds__(256)
bn_bwd_apply_kernel(const float* __restrict__ G, int ldg, const float* __restrict__ Y, int ldy,
                    const float* __restrict__ scale, const float* __restrict__ shift, const float* __restrict__ mean,
                    const float* __restrict__ invstd, const float* __restrict__ c1, const float* __restrict__ c2,
                    int relu, float* __restrict__ GY, int ldo, int P, int C) {
  const int c4n = C >> 2, rpp = 256 / c4n;
  const int c = (threadIdx.x % c4n) * 4, rl = threadIdx.x / c4n;
  const float4 sc = *reinterpret_cast<const float4*>(scale + c), sh = *reinterpret_cast<const float4*>(shift + c);
  const float4 mu = *reinterpret_cast<const float4*>(mean + c), is = *reinterpret_cast<const float4*>(invstd + c);
  const float4 k1 = *reinterpret_cast<const float4*>(c1 + c), k2 = *reinterpret_cast<const float4*>(c2 + c);
  const float scv[4] = {sc.x, sc.y, sc.z, sc.w}, shv[4] = {sh.x, sh.y, sh.z, sh.w}, muv[4] = {mu.x, mu.y, mu.z, mu.w};
  const float isv[4] = {is.x, is.y, is.z, is.w}, k1v[4] = {k1.x, k1.y, k1.z, k1.w}, k2v[4] = {k2.x, k2.y, k2.z, k2.w};
  const long long step = (long long)gridDim.x * rpp;
  for (long long r0 = (long long)blockIdx.x * rpp + rl; r0 < P; r0 += 4 * step) {
    float4 g4[4], y4[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const long long r = r0 + u * step;
      if (r < P) {
        g4[u] = __ldcs(reinterpret_cast<const float4*>(G + (size_t)r * ldg + c));
        y4[u] = __ldcs(reinterpret_cast<const float4*>(Y + (size_t)r * ldy + c));
      }
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const long long r = r0 + u * step;
      if (r < P) {
        const float gv[4] = {g4[u].x, g4[u].y, g4[u].z, g4[u].w}, yv[4] = {y4[u].x, y4[u].y, y4[u].z, y4[u].w};
        float o[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float z = fmaf(yv[j], scv[j], shv[j]);
          const float gz = (!relu || z > 0.f) ? gv[j] : 0.f;
          o[j] = scv[j] * (gz - k1v[j] - (yv[j] - muv[j]) * isv[j] * k2v[j]);
        }
        *reinterpret_cast<float4*>(GY + (size_t)r * ldo + c) = make_float4(o[0], o[1], o[2], o[3]);
      }
    }
  }
}
// any C % 4 == 0: grid-stride over (row, 4-column group)
__global__ void __launch_bounds__(256)
bn_bwd_apply_generic_kernel(const float* __restrict__ G, int ldg, const float* __restrict__ Y, int ldy,
                            const float* __restrict__ scale, const float* __restrict__ shift, const float* __restrict__ mean,
                            const float* __restrict__ invstd, const float* __restrict__ c1, const float* __restrict__ c2,
                            int relu, float* __restrict__ GY, int ldo, int P, int C) {
  const int c4n = C / 4;
  const size_t total = (size_t)P * c4n;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int r = (int)(i / c4n), c = (int)(i - (size_t)r * c4n) * 4;
    const float4 g4 = *reinterpret_cast<const float4*>(G + (size_t)r * ldg + c);
    const float4 y4 = *reinterpret_cast<const float4*>(Y + (size_t)r * ldy + c);
    const float gv[4] = {g4.x, g4.y, g4.z, g4.w}, yv[4] = {y4.x, y4.y, y4.z, y4.w};
    float o[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float sc = scale[c + j];
      const float z = fmaf(yv[j], sc, shift[c + j]);
      const float gz = (!relu || z > 0.f) ? gv[j] : 0.f;
      o[j] = sc * (gz - c1[c + j] - (yv[j] - mean[c + j]) * invstd[c + j] * c2[c + j]);
    }
    *reinterpret_cast<float4*>(GY + (size_t)r * ldo + c) = make_float4(o[0], o[1], o[2], o[3]);
  }
}

// ------------------------------------------------------------------------------------------------
// group-max layers: out[q,c] = relu(scale*ysel+shift), ysel = (scale>=0 ? gmax : gmin)[q,c] at row arg.
//   select : gz[q,c] = g_out[q,c]*1[z>0], argsel[q,c]; partial sums of gz and gz*xhat(ysel) over q tiles
//   scatter: G[(q*K+argsel), c] += gz_or_g[q,c]            (max path joins a dense gradient)
//   apply  : g_y[(q,k),c] = scale*( (k==argsel)*gz - c1 - xhat*c2 )   (max is the ONLY consumer)
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
groupmax_bwd_select_kernel(const float* __restrict__ Gout, int ldg, const float* __restrict__ gmax,
                           const float* __restrict__ gmin, const int32_t* __restrict__ amax,
                           const int32_t* __restrict__ amin, const float* __restrict__ scale,
                           const float* __restrict__ shift, const float* __restrict__ mean,
                           const float* __restrict__ invstd, float* __restrict__ gz, int32_t* __restrict__ argsel,
                           float* __restrict__ part, int Q, int C) {
  // CTA = 128 q-rows x 32 channels, thread = (row slice of 8, channel): 4x the CTAs of the 128-channel tiling (the
  // 8192 x 512 head only made 256 CTAs, each thread walking 64 rows in turn -- 70 us of exposed load latency)
  __shared__ float red[2][8][32];
  const int tile = blockIdx.x, cl = threadIdx.x & 31, c = blockIdx.y * 32 + cl, rs = threadIdx.x >> 5;
  float s1 = 0.f, s2 = 0.f;
  if (c < C) {
    const float sc = scale[c], sh = shift[c], mu = mean ? mean[c] : 0.f, is = invstd ? invstd[c] : 0.f;
    const bool up = sc >= 0.f;
    const float* __restrict__ ysrc = up ? gmax : gmin;
    const int32_t* __restrict__ asrc = up ? amax : amin;
    const int qend = min(Q, (tile + 1) * BW_ROWS);
#pragma unroll 4
    for (int q = tile * BW_ROWS + rs; q < qend; q += 8) {
      const size_t i = (size_t)q * C + c;
      const float ys = ysrc[i];
      const float go = Gout[(size_t)q * ldg + c];
      const int a = asrc[i];
      const float g = fmaf(ys, sc, sh) > 0.f ? go : 0.f;
      gz[i] = g; argsel[i] = a;
      s1 += g; s2 = fmaf(g, (ys - mu) * is, s2);
    }
  }
  red[0][rs][cl] = s1; red[1][rs][cl] = s2;
  __syncthreads();
  if (part && threadIdx.x < 32 && c < C) {
    float a = 0.f, b = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) { a += red[0][j][cl]; b += red[1][j][cl]; }
    part[((size_t)tile * 2 + 0) * C + c] = a;
    part[((size_t)tile * 2 + 1) * C + c] = b;
  }
}

__global__ void groupmax_scatter_add_kernel(float* __restrict__ G, int ldg, const float* __restrict__ gsrc,
                                            const int32_t* __restrict__ argsel, int K, int Q, int C) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)Q * C) return;
  int q = (int)(i / C), c = (int)(i - (size_t)q * C);
  G[((size_t)q * K + argsel[i]) * ldg + c] += gsrc[i];        // unique target per (q,c): no atomics needed
}

__global__ void __launch_bounds__(256)
groupmax_bwd_apply_kernel(const float* __restrict__ Y, int ldy, const float* __restrict__ gz,
                          const int32_t* __restrict__ argsel, const float* __restrict__ scale,
                          const float* __restrict__ mean, const float* __restrict__ invstd,
                          const float* __restrict__ c1, const float* __restrict__ c2, float* __restrict__ GY, int ldo,
                          int K, int P, int C) {
  const int c4n = C / 4;
  const size_t total = (size_t)P * c4n;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int r = (int)(i / c4n), c = (int)(i - (size_t)r * c4n) * 4;
    const int q = r / K, k = r - q * K;
    const float4 y4 = *reinterpret_cast<const float4*>(Y + (size_t)r * ldy + c);
    const float4 g4 = *reinterpret_cast<const float4*>(gz + (size_t)q * C + c);
    const int4 a4 = *reinterpret_cast<const int4*>(argsel + (size_t)q * C + c);
    const float yv[4] = {y4.x, y4.y, y4.z, y4.w}, gv[4] = {g4.x, g4.y, g4.z, g4.w};
    const int av[4] = {a4.x, a4.y, a4.z, a4.w};
    // per-channel constants as five 16-byte loads (they were twenty scalar loads: the LSU queue was the top stall)
    const float4 s4 = __ldg(reinterpret_cast<const float4*>(scale + c)), m4 = __ldg(reinterpret_cast<const float4*>(mean + c));
    const float4 i4 = __ldg(reinterpret_cast<const float4*>(invstd + c)), p4 = __ldg(reinterpret_cast<const float4*>(c1 + c));
    const float4 q4 = __ldg(reinterpret_cast<const float4*>(c2 + c));
    const float sv[4] = {s4.x, s4.y, s4.z, s4.w}, mv[4] = {m4.x, m4.y, m4.z, m4.w}, iv[4] = {i4.x, i4.y, i4.z, i4.w};
    const float c1v[4] = {p4.x, p4.y, p4.z, p4.w}, c2v[4] = {q4.x, q4.y, q4.z, q4.w};
    float o[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float g = (av[j] == k) ? gv[j] : 0.f;
      o[j] = sv[j] * (g - c1v[j] - (yv[j] - mv[j]) * iv[j] * c2v[j]);
    }
    *reinterpret_cast<float4*>(GY + (size_t)r * ldo + c) = make_float4(o[0], o[1], o[2], o[3]);
  }
}

// out[q,c] = sum_k G[(q*K+k), c]
__global__ void group_sum_kernel(const float* __restrict__ G, int ldg, float* __restrict__ out, int ldo, int K, int Q,
                                 int C) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int c4n = C / 4;
  if (i >= (size_t)Q * c4n) return;
  int q = (int)(i / c4n), c = (int)(i - (size_t)q * c4n) * 4;
  float4 s = make_float4(0, 0, 0, 0);
  for (int k = 0; k < K; ++k) {
    float4 v = *reinterpret_cast<const float4*>(G + ((size_t)q * K + k) * ldg + c);
    s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
  }
  *reinterpret_cast<float4*>(out + (size_t)q * ldo + c) = s;
}

// out[seg,c] = sum over the contiguous rows of the segment (warp per segment)
__global__ void __launch_bounds__(256)
seg_sum_kernel(const float* __restrict__ G, int ldg, const int32_t* __restrict__ seg_off, float* __restrict__ out,
               int ldo, int B, int N, int M, int C) {
  const int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (w >= B * M) return;
  const int b = w / M, m = w - b * M;
  const int s = seg_off[(size_t)b * (M + 1) + m], e = seg_off[(size_t)b * (M + 1) + m + 1];
  for (int c4 = lane; c4 * 4 < C; c4 += 32) {
    float4 a = make_float4(0, 0, 0, 0);
    for (int r = s; r < e; ++r) {
      float4 v = *reinterpret_cast<const float4*>(G + ((size_t)b * N + r) * ldg + c4 * 4);
      a.x += v.x; a.y += v.y; a.z += v.z; a.w += v.w;
    }
    *reinterpret_cast<float4*>(out + (size_t)w * ldo + c4 * 4) = a;
  }
}

// arg-max un-pooling: G[arg[q,c], c] (+)= gp[q,c]; arg = global row or -1 (empty node)
__global__ void unpool_scatter_kernel(float* __restrict__ G, int ldg, const float* __restrict__ gp, int ldp,
                                      const int32_t* __restrict__ arg, int Q, int C, int accumulate) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)Q * C) return;
  int q = (int)(i / C), c = (int)(i - (size_t)q * C);
  int r = arg[i];
  if (r < 0) return;
  float v = gp[(size_t)q * ldp + c];
  float* dst = G + (size_t)r * ldg + c;
  *dst = accumulate ? *dst + v : v;                          // targets are unique per (q,c)
}

// backward of usip_knn_combine: G_Z[b*M+nbr] += GY[row]; gWxyz[c,0..2] += GY[row,c]*delta
__global__ void __launch_bounds__(256)
knn_combine_bwd_kernel(const float* __restrict__ GY, int ldg, const float* __restrict__ pts,
                       const int32_t* __restrict__ knn_idx, float* __restrict__ GZ, int ldz, float* __restrict__ gW,
                       int ldw, int B, int M, int K, int C) {
  extern __shared__ float sw[];                              // [C][3]
  for (int i = threadIdx.x; i < C * 3; i += 256) sw[i] = 0.f;
  __syncthreads();
  const int row0 = blockIdx.x * BW_ROWS, G = B * M * K;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const bool vec = (ldz % 4 == 0) && ((reinterpret_cast<uintptr_t>(GZ) & 15) == 0);
  for (int c4 = lane; c4 * 4 < C; c4 += 32) {
    float a0[4] = {0, 0, 0, 0}, a1[4] = {0, 0, 0, 0}, a2[4] = {0, 0, 0, 0};
    for (int r = row0 + warp; r < min(row0 + BW_ROWS, G); r += 8) {
      const int q = r / K, b = q / M, m = q - b * M, j = knn_idx[r];
      const float* p = pts + (size_t)b * 3 * M;
      const float dx = p[j] - p[m], dy = p[M + j] - p[M + m], dz = p[2 * M + j] - p[2 * M + m];
      const float4 g = *reinterpret_cast<const float4*>(GY + (size_t)r * ldg + c4 * 4);
      const float gv[4] = {g.x, g.y, g.z, g.w};
      float* z = GZ + ((size_t)b * M + j) * ldz + c4 * 4;
      if (vec) {                                             // one 16-byte L2 reduction instead of four (sm_90+)
        atomicAdd(reinterpret_cast<float4*>(z), g);
      } else {
#pragma unroll
        for (int t = 0; t < 4; ++t) atomicAdd(z + t, gv[t]);
      }
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        a0[t] = fmaf(gv[t], dx, a0[t]); a1[t] = fmaf(gv[t], dy, a1[t]); a2[t] = fmaf(gv[t], dz, a2[t]);
      }
    }
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      atomicAdd(&sw[(c4 * 4 + t) * 3 + 0], a0[t]); atomicAdd(&sw[(c4 * 4 + t) * 3 + 1], a1[t]);
      atomicAdd(&sw[(c4 * 4 + t) * 3 + 2], a2[t]);
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < C * 3; i += 256) atomicAdd(&gW[(size_t)(i / 3) * ldw + (i % 3)], sw[i]);
}

// column sums: out[c] += sum_r G[r,c].  HBM-bound ([262144 x 128] fp32 = 134 MB): every thread streams float4s of one
// 4-column group over a strided set of rows (a warp covers 128 consecutive floats of a row when C >= 128, whole rows
// otherwise), partial sums meet in shared memory, one atomicAdd per column and CTA.
__global__ void __launch_bounds__(256)
colsum_kernel(const float* __restrict__ G, int ldg, float* __restrict__ out, int P, int C) {
  __shared__ float red[256][4];
  const int c4n = C >> 2;                                   // float4 groups per row (host guarantees C % 4 == 0, C <= 1024)
  const int cg = threadIdx.x % c4n, rl = threadIdx.x / c4n, rpp = 256 / c4n;   // rows per pass of this CTA
  float s[4] = {0.f, 0.f, 0.f, 0.f};
  if (rl < rpp) {
    for (long long r = (long long)blockIdx.x * rpp + rl; r < P; r += (long long)gridDim.x * rpp) {
      const float4 v = __ldcs(reinterpret_cast<const float4*>(G + (size_t)r * ldg + cg * 4));
      s[0] += v.x; s[1] += v.y; s[2] += v.z; s[3] += v.w;
    }
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) red[threadIdx.x][j] = s[j];
  __syncthreads();
  if (threadIdx.x < c4n) {
    float t[4] = {0.f, 0.f, 0.f, 0.f};
    for (int k = 0; k < rpp; ++k)
#pragma unroll
      for (int j = 0; j < 4; ++j) t[j] += red[k * c4n + threadIdx.x][j];
#pragma unroll
    for (int j = 0; j < 4; ++j) atomicAdd(out + threadIdx.x * 4 + j, t[j]);
  }
}
// generic fallback (any C, any alignment): one thread per column over a 1024-row slab
__global__ void __launch_bounds__(256)
colsum_slow_kernel(const float* __restrict__ G, int ldg, float* __restrict__ out, int P, int C) {
  const int c = blockIdx.y * 256 + threadIdx.x;
  if (c >= C) return;
  const int r0 = blockIdx.x * 1024, r1 = min(P, r0 + 1024);
  float s = 0.f;
  for (int r = r0; r < r1; ++r) s += G[(size_t)r * ldg + c];
  atomicAdd(out + c, s);
}

// wgrad for a NARROW input (Cin <= 8, e.g. the first layer of a point stack: xyz + normals):
//   gW[m, j] += sum_r GY[r, m] * act(X)[r, j].   HBM-bound on GY ([P, Cout] read once).  Thread = FOUR output channels of
// one row subset (one 16-byte GY load per row, 4 x 8 accumulators); the X row is a 32-byte broadcast shared by the Cout/4
// threads of the row and its activation is computed once per thread and row.  (Round 2, first version: one channel per
// thread = one 4-byte load and 30 instructions per GY element, 137 us for the 262144 x 64 first layer = 0.55 TB/s.)
__global__ void __launch_bounds__(256, 2)
wgrad_narrow_kernel(const float* __restrict__ GY, int ldg, const float* __restrict__ X, int ldx,
                    const float* __restrict__ in_scale, const float* __restrict__ in_shift, int in_relu,
                    float* __restrict__ gW, int ldw, int P, int Cout, int Cin) {
  __shared__ float red[256][33];
  const int tpr = Cout >> 2, rpp = 256 / tpr;                  // host: Cout in {32, 64, 128, 256}
  const int c4 = threadIdx.x % tpr, rl = threadIdx.x / tpr;
  float acc[4][8];
#pragma unroll
  for (int q = 0; q < 4; ++q)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[q][j] = 0.f;
  float sc[8], sh[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) { sc[j] = (in_scale && j < Cin) ? in_scale[j] : 1.f; sh[j] = (in_shift && j < Cin) ? in_shift[j] : 0.f; }
  const bool x8 = (ldx == 8) && ((reinterpret_cast<uintptr_t>(X) & 15) == 0);
  const long long step = (long long)gridDim.x * rpp;
  for (long long r0 = (long long)blockIdx.x * rpp + rl; r0 < P; r0 += 4 * step) {
    float4 g[4], xa[4], xb[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {                              // four independent rows in flight per thread
      const long long r = r0 + u * step;
      g[u] = xa[u] = xb[u] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (r < P) {
        g[u] = __ldcs(reinterpret_cast<const float4*>(GY + (size_t)r * ldg + c4 * 4));
        if (x8) {
          xa[u] = __ldg(reinterpret_cast<const float4*>(X + (size_t)r * 8)); xb[u] = __ldg(reinterpret_cast<const float4*>(X + (size_t)r * 8 + 4));
        } else {
          float t[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
          for (int j = 0; j < Cin; ++j) t[j] = __ldg(X + (size_t)r * ldx + j);
          xa[u] = make_float4(t[0], t[1], t[2], t[3]); xb[u] = make_float4(t[4], t[5], t[6], t[7]);
        }
      }
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const float x[8] = {xa[u].x, xa[u].y, xa[u].z, xa[u].w, xb[u].x, xb[u].y, xb[u].z, xb[u].w};
      const float gq[4] = {g[u].x, g[u].y, g[u].z, g[u].w};   // rows past P carry g = 0
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        float v = fmaf(x[j], sc[j], sh[j]);
        if (in_relu) v = fmaxf(v, 0.f);
        v = j < Cin ? v : 0.f;
#pragma unroll
        for (int q = 0; q < 4; ++q) acc[q][j] = fmaf(gq[q], v, acc[q][j]);
      }
    }
  }
#pragma unroll
  for (int q = 0; q < 4; ++q)
#pragma unroll
    for (int j = 0; j < 8; ++j) red[threadIdx.x][q * 8 + j] = acc[q][j];
  __syncthreads();
  for (int i = threadIdx.x; i < Cout * Cin; i += 256) {
    const int m = i / Cin, j = i - m * Cin;
    float t = 0.f;
    for (int k = 0; k < rpp; ++k) t += red[k * tpr + (m >> 2)][(m & 3) * 8 + j];
    atomicAdd(gW + (size_t)m * ldw + j, t);
  }
}

// networks.py:151-154 backward: G_out4[q,0:3] = g_kp, G_out4[q,3] = g_sig * sigmoid(x)
__global__ void head_bwd_kernel(const float* __restrict__ g_kp, const float* __restrict__ g_sig,
                                const float* __restrict__ out4, int ld, float* __restrict__ G, int B, int M) {
  int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= B * M) return;
  int b = t / M, m = t - b * M;
  float4 o;
  o.x = g_kp ? g_kp[(size_t)b * 3 * M + m] : 0.f;
  o.y = g_kp ? g_kp[(size_t)b * 3 * M + M + m] : 0.f;
  o.z = g_kp ? g_kp[(size_t)b * 3 * M + 2 * M + m] : 0.f;
  float x = out4[(size_t)t * ld + 3];
  float ds = x > 20.f ? 1.f : 1.f / (1.f + expf(-x));
  o.w = g_sig ? g_sig[t] * ds : 0.f;
  *reinterpret_cast<float4*>(G + (size_t)t * 4) = o;
}

// ------------------------------------------------------------------------------------------------
// wgrad: gW[Cout,Cin] += GY[P,Cout]^T * act(X)[P,Cin]   (split over row ranges, atomic accumulation)
// ------------------------------------------------------------------------------------------------
constexpr int WG_BK = 16;
constexpr int WG_LD = 128 + 4;

__global__ void __launch_bounds__(256, 2)
wgrad_simt_kernel(const float* __restrict__ GY, int ldg, const float* __restrict__ X, int ldx,
                  const float* __restrict__ in_scale, const float* __restrict__ in_shift, int in_relu,
                  float* __restrict__ gW, int ldw, int P, int Cout, int Cin, int rows_per_cta) {
  __shared__ __align__(16) float As[2][WG_BK][WG_LD];
  __shared__ __align__(16) float Bs[2][WG_BK][WG_LD];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int m0 = blockIdx.y * 128, n0 = blockIdx.z * 128;       // m: Cout index, n: Cin index
  const int r_begin = blockIdx.x * rows_per_cta, r_end = min(P, r_begin + rows_per_cta);
  const int lk = tid >> 5, l4 = tid & 31;                        // row-in-chunk (0..7, +8), float4 column
  const bool a_vec = ((ldg & 3) == 0) && ((reinterpret_cast<uintptr_t>(GY) & 15) == 0);
  const bool b_vec = ((ldx & 3) == 0) && ((reinterpret_cast<uintptr_t>(X) & 15) == 0);
  float4 sc = make_float4(1, 1, 1, 1), sh = make_float4(0, 0, 0, 0);
  const int bc = n0 + l4 * 4;
  if (in_scale) {
    float s[4], h[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) { s[j] = bc + j < Cin ? in_scale[bc + j] : 0.f; h[j] = bc + j < Cin ? in_shift[bc + j] : 0.f; }
    sc = make_float4(s[0], s[1], s[2], s[3]); sh = make_float4(h[0], h[1], h[2], h[3]);
  }
  float4 ar[2], br[2];
  auto load = [&](int r0) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = r0 + lk + 8 * h;
      const int ac = m0 + l4 * 4;
      float a[4] = {0, 0, 0, 0}, b[4] = {0, 0, 0, 0};
      if (r < r_end) {
        if (a_vec && ac + 4 <= Cout) { float4 v = *reinterpret_cast<const float4*>(GY + (size_t)r * ldg + ac); a[0] = v.x; a[1] = v.y; a[2] = v.z; a[3] = v.w; }
        else { for (int j = 0; j < 4; ++j) if (ac + j < Cout) a[j] = GY[(size_t)r * ldg + ac + j]; }
        if (b_vec && bc + 4 <= Cin) { float4 v = *reinterpret_cast<const float4*>(X + (size_t)r * ldx + bc); b[0] = v.x; b[1] = v.y; b[2] = v.z; b[3] = v.w; }
        else { for (int j = 0; j < 4; ++j) if (bc + j < Cin) b[j] = X[(size_t)r * ldx + bc + j]; }
        if (in_scale) { b[0] = fmaf(b[0], sc.x, sh.x); b[1] = fmaf(b[1], sc.y, sh.y); b[2] = fmaf(b[2], sc.z, sh.z); b[3] = fmaf(b[3], sc.w, sh.w); }
        if (in_relu) { b[0] = fmaxf(b[0], 0.f); b[1] = fmaxf(b[1], 0.f); b[2] = fmaxf(b[2], 0.f); b[3] = fmaxf(b[3], 0.f); }
#pragma unroll
        for (int j = 0; j < 4; ++j) if (bc + j >= Cin) b[j] = 0.f;
      }
      ar[h] = make_float4(a[0], a[1], a[2], a[3]); br[h] = make_float4(b[0], b[1], b[2], b[3]);
    }
  };
  auto store = [&](int buf) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      *reinterpret_cast<float4*>(&As[buf][lk + 8 * h][l4 * 4]) = ar[h];
      *reinterpret_cast<float4*>(&Bs[buf][lk + 8 * h][l4 * 4]) = br[h];
    }
  };
  float acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
  const int nchunks = (r_end - r_begin + WG_BK - 1) / WG_BK;
  if (nchunks <= 0) return;
  load(r_begin); store(0);
  __syncthreads();
  for (int ch = 0; ch < nchunks; ++ch) {
    const int buf = ch & 1;
    if (ch + 1 < nchunks) load(r_begin + (ch + 1) * WG_BK);
#pragma unroll
    for (int k = 0; k < WG_BK; ++k) {
      const float4 a0 = *reinterpret_cast<const float4*>(&As[buf][k][ty * 4]);
      const float4 a1 = *reinterpret_cast<const float4*>(&As[buf][k][64 + ty * 4]);
      const float4 b0 = *reinterpret_cast<const float4*>(&Bs[buf][k][tx * 4]);
      const float4 b1 = *reinterpret_cast<const float4*>(&Bs[buf][k][64 + tx * 4]);
      const float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      const float b[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    if (ch + 1 < nchunks) store(buf ^ 1);
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int m = m0 + (i < 4 ? ty * 4 + i : 64 + ty * 4 + (i - 4));
    if (m >= Cout) continue;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int n = n0 + (j < 4 ? tx * 4 + j : 64 + tx * 4 + (j - 4));
      if (n < Cin) atomicAdd(gW + (size_t)m * ldw + n, acc[i][j]);
    }
  }
}


// backward of descriptor / (||descriptor|| + 1e-5) (networks.py:383): g (B,C,M) reference layout, y raw rows [Q,C]
//   out = y / (n + eps):  g_y = g / (n + eps) - y * (g . y) / (n * (n + eps)^2)      (n = 0: torch.norm's sub-gradient is 0)
__global__ void __launch_bounds__(256)
l2norm_bwd_kernel(const float* __restrict__ g, const float* __restrict__ Y, int ldy, float* __restrict__ GY, int ldg,
                  int B, int M, int C) {
  const int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (w >= B * M) return;
  const int b = w / M, m = w - b * M;
  const float* y = Y + (size_t)w * ldy;
  float ss = 0.f, gy = 0.f;
  for (int c = lane; c < C; c += 32) {
    const float yv = y[c], gv = g[((size_t)b * C + c) * M + m];
    ss = fmaf(yv, yv, ss); gy = fmaf(gv, yv, gy);
  }
  ss = warp_sum(ss); gy = warp_sum(gy);
  const float n = sqrtf(ss), d = n + 1e-5f;
  const float k = n > 0.f ? gy / (n * d * d) : 0.f;
  for (int c = lane; c < C; c += 32) GY[(size_t)w * ldg + c] = g[((size_t)b * C + c) * M + m] / d - y[c] * k;
}

// backward of DescPairScanLoss (losses.py:199-233): loss[b,m] = w * clamp(dpos - dneg + gamma, 0) with upstream gradient
// g_loss (B,M).  Thread block = one (b, m): coef = g_loss * w where the hinge is active; the anchor receives
// coef * ((a - p)/dpos - (a - n)/dneg), the matched positive -coef*(a - p)/dpos and the matched negative +coef*(a - n)/dneg
// (scattered with atomics: several anchors can share a match).  The weights are detached in the reference.
__global__ void __launch_bounds__(128)
desc_triplet_bwd_kernel(const float* __restrict__ anc, const float* __restrict__ pos, const float* __restrict__ neg,
                        const float* __restrict__ dpos, const int32_t* __restrict__ ipos, const float* __restrict__ dneg,
                        const int32_t* __restrict__ ineg, const float* __restrict__ sigma, float gamma, float sigma_max,
                        const float* __restrict__ g_loss, float* __restrict__ g_anc, float* __restrict__ g_pos,
                        float* __restrict__ g_neg, int C, int M, int Mp, int Mn) {
  __shared__ float s_wmean;
  __shared__ float sred[4];
  const int b = blockIdx.y, m = blockIdx.x;
  float ws = 0.f;
  for (int t = threadIdx.x; t < M; t += blockDim.x) ws += fmaxf(sigma_max - sigma[(size_t)b * M + t], 0.f);
  ws = warp_sum(ws);
  if ((threadIdx.x & 31) == 0) sred[threadIdx.x >> 5] = ws;
  __syncthreads();
  if (threadIdx.x == 0) s_wmean = (sred[0] + sred[1] + sred[2] + sred[3]) / (float)M;
  __syncthreads();
  const size_t bm = (size_t)b * M + m;
  const float dp = dpos[bm], dn = dneg[bm];
  if (!(dp - dn + gamma > 0.f)) return;
  const float coef = g_loss[bm] * (fmaxf(sigma_max - sigma[bm], 0.f) / s_wmean);
  const int jp = ipos[bm], jn = ineg[bm];
  const float ip = dp > 0.f ? coef / dp : 0.f, in = dn > 0.f ? coef / dn : 0.f;      // torch.norm: zero sub-gradient at 0
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    const float a = anc[((size_t)b * C + c) * M + m];
    const float tp = (a - pos[((size_t)b * C + c) * Mp + jp]) * ip;
    const float tn = (a - neg[((size_t)b * C + c) * Mn + jn]) * in;
    atomicAdd(&g_anc[((size_t)b * C + c) * M + m], tp - tn);
    atomicAdd(&g_pos[((size_t)b * C + c) * Mp + jp], -tp);
    atomicAdd(&g_neg[((size_t)b * C + c) * Mn + jn], tn);
  }
}

}  // namespace usip

using namespace usip;

extern "C" int usip_bn_bwd_reduce(const float* G, int ldg, const float* Y, int ldy, const float* scale,
                                  const float* shift, const float* mean, const float* invstd, int relu,
                                  float* part, int P, int C, void* stream) {
  USIP_REQUIRE(G && Y && scale && shift && mean && invstd && part && C % 4 == 0 && ldg % 4 == 0 && ldy % 4 == 0 &&
               (C <= 128 ? (128 % C == 0 || C % 4 == 0) : C % 128 == 0), "bn_bwd_reduce: bad args");
  USIP_REQUIRE(C >= 32, "bn_bwd_reduce: C must be >= 32");
  // both kernels read G, Y and the per-channel vectors as float4 (the fast one also writes part as float4)
  USIP_REQUIRE(((reinterpret_cast<uintptr_t>(G) | reinterpret_cast<uintptr_t>(Y) | reinterpret_cast<uintptr_t>(part) |
                 reinterpret_cast<uintptr_t>(scale) | reinterpret_cast<uintptr_t>(shift) | reinterpret_cast<uintptr_t>(mean) |
                 reinterpret_cast<uintptr_t>(invstd)) & 15) == 0,
               "bn_bwd_reduce: operands must be 16-byte aligned");
  const int c4n = C / 4, ntiles = cdiv(P, BW_ROWS);
  if (c4n <= 256 && 256 % c4n == 0) {
    const int blocks = min(ntiles, device_sm_count() * 4);
    bn_bwd_reduce_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(G, ldg, Y, ldy, scale, shift, mean, invstd, relu, part, P, C, ntiles);
    return check_launch("bn_bwd_reduce_kernel");
  }
  dim3 grid(cdiv(P, BW_ROWS), cdiv(C, 128));
  bn_bwd_reduce_tile_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(G, ldg, Y, ldy, scale, shift, mean, invstd, relu, part, P, C);
  return check_launch("bn_bwd_reduce_kernel");
}

extern "C" int usip_bn_bwd_finalize(const float* part, int ntiles, int64_t count, int C, float* g_gamma, float* g_beta,
                                    float* c1, float* c2, int accumulate, void* stream) {
  USIP_REQUIRE(part && c1 && c2 && ntiles > 0, "bn_bwd_finalize: bad args");
  bn_bwd_finalize_kernel<<<cdiv(C, 8), 256, 0, (cudaStream_t)stream>>>(part, ntiles, (double)count, C, g_gamma, g_beta,
                                                                         c1, c2, accumulate);
  return check_launch("bn_bwd_finalize_kernel");
}

extern "C" int usip_bn_bwd_apply(const float* G, int ldg, const float* Y, int ldy, const float* scale, const float* shift,
                                 const float* mean, const float* invstd, const float* c1, const float* c2, int relu,
                                 float* GY, int ldo, int P, int C, void* stream) {
  USIP_REQUIRE(G && Y && GY && scale && shift && mean && invstd && c1 && c2 && C % 4 == 0 && ldg % 4 == 0 &&
               ldy % 4 == 0 && ldo % 4 == 0, "bn_bwd_apply: bad args");
  // G, Y, GY are float4 rows in both kernels; the fast one also reads the per-channel vectors as float4
  USIP_REQUIRE(((reinterpret_cast<uintptr_t>(G) | reinterpret_cast<uintptr_t>(Y) | reinterpret_cast<uintptr_t>(GY) |
                 reinterpret_cast<uintptr_t>(scale) | reinterpret_cast<uintptr_t>(shift) | reinterpret_cast<uintptr_t>(mean) |
                 reinterpret_cast<uintptr_t>(invstd) | reinterpret_cast<uintptr_t>(c1) | reinterpret_cast<uintptr_t>(c2)) & 15) == 0,
               "bn_bwd_apply: operands must be 16-byte aligned");
  size_t total = (size_t)P * (C / 4);
  const int c4n = C / 4;
  if (c4n <= 256 && 256 % c4n == 0) {
    const int rpp = 256 / c4n;
    const int blocks = (int)min((long long)device_sm_count() * 8, (long long)cdiv(P, rpp * 4));
    bn_bwd_apply_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(G, ldg, Y, ldy, scale, shift, mean, invstd, c1, c2, relu, GY, ldo, P, C);
    return check_launch("bn_bwd_apply_kernel");
  }
  int blocks = (int)min((size_t)device_sm_count() * 16, cdiv64(total, 256));
  bn_bwd_apply_generic_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(G, ldg, Y, ldy, scale, shift, mean, invstd, c1, c2, relu,
                                                                        GY, ldo, P, C);
  return check_launch("bn_bwd_apply_generic_kernel");
}

extern "C" int usip_groupmax_bwd_select(const float* Gout, int ldg, const float* gmax, const float* gmin,
                                        const int32_t* amax, const int32_t* amin, const float* scale,
                                        const float* shift, const float* mean, const float* invstd, float* gz,
                                        int32_t* argsel, float* part, int Q, int C, void* stream) {
  USIP_REQUIRE(Gout && gmax && gmin && amax && amin && scale && shift && gz && argsel, "groupmax_bwd_select: bad args");
  dim3 grid(cdiv(Q, BW_ROWS), cdiv(C, 32));
  groupmax_bwd_select_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(Gout, ldg, gmax, gmin, amax, amin, scale, shift, mean,
                                                                     invstd, gz, argsel, part, Q, C);
  return check_launch("groupmax_bwd_select_kernel");
}

extern "C" int usip_groupmax_scatter_add(float* G, int ldg, const float* gsrc, const int32_t* argsel, int K, int Q,
                                         int C, void* stream) {
  USIP_REQUIRE(G && gsrc && argsel, "groupmax_scatter_add: bad args");
  size_t n = (size_t)Q * C;
  groupmax_scatter_add_kernel<<<(unsigned)cdiv64(n, 256), 256, 0, (cudaStream_t)stream>>>(G, ldg, gsrc, argsel, K, Q, C);
  return check_launch("groupmax_scatter_add_kernel");
}

extern "C" int usip_groupmax_bwd_apply(const float* Y, int ldy, const float* gz, const int32_t* argsel,
                                       const float* scale, const float* mean, const float* invstd, const float* c1,
                                       const float* c2, float* GY, int ldo, int K, int P, int C, void* stream) {
  USIP_REQUIRE(Y && gz && argsel && GY && C % 4 == 0 && ldy % 4 == 0 && ldo % 4 == 0, "groupmax_bwd_apply: bad args");
  USIP_REQUIRE(((reinterpret_cast<uintptr_t>(Y) | reinterpret_cast<uintptr_t>(gz) | reinterpret_cast<uintptr_t>(argsel) |
                 reinterpret_cast<uintptr_t>(GY) | reinterpret_cast<uintptr_t>(scale) | reinterpret_cast<uintptr_t>(mean) |
                 reinterpret_cast<uintptr_t>(invstd) | reinterpret_cast<uintptr_t>(c1) | reinterpret_cast<uintptr_t>(c2)) & 15) == 0,
               "groupmax_bwd_apply: operands must be 16-byte aligned");
  size_t total = (size_t)P * (C / 4);
  int blocks = (int)min((size_t)device_sm_count() * 16, cdiv64(total, 256));
  groupmax_bwd_apply_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(Y, ldy, gz, argsel, scale, mean, invstd, c1, c2, GY,
                                                                      ldo, K, P, C);
  return check_launch("groupmax_bwd_apply_kernel");
}

extern "C" int usip_group_sum(const float* G, int ldg, float* out, int ldo, int K, int Q, int C, void* stream) {
  USIP_REQUIRE(G && out && C % 4 == 0 && ldg % 4 == 0 && ldo % 4 == 0, "group_sum: bad args");
  USIP_REQUIRE(((reinterpret_cast<uintptr_t>(G) | reinterpret_cast<uintptr_t>(out)) & 15) == 0,
               "group_sum: G and out must be 16-byte aligned");
  size_t n = (size_t)Q * (C / 4);
  group_sum_kernel<<<(unsigned)cdiv64(n, 256), 256, 0, (cudaStream_t)stream>>>(G, ldg, out, ldo, K, Q, C);
  return check_launch("group_sum_kernel");
}

extern "C" int usip_seg_sum(const float* G, int ldg, const int32_t* seg_off, float* out, int ldo, int B, int N, int M,
                            int C, void* stream) {
  USIP_REQUIRE(G && seg_off && out && C % 4 == 0 && ldg % 4 == 0 && ldo % 4 == 0, "seg_sum: bad args");
  USIP_REQUIRE(((reinterpret_cast<uintptr_t>(G) | reinterpret_cast<uintptr_t>(out)) & 15) == 0,
               "seg_sum: G and out must be 16-byte aligned");
  seg_sum_kernel<<<cdiv(B * M * 32, 256), 256, 0, (cudaStream_t)stream>>>(G, ldg, seg_off, out, ldo, B, N, M, C);
  return check_launch("seg_sum_kernel");
}

extern "C" int usip_unpool_scatter(float* G, int ldg, const float* gp, int ldp, const int32_t* arg, int Q, int C,
                                   int accumulate, void* stream) {
  USIP_REQUIRE(G && gp && arg, "unpool_scatter: bad args");
  size_t n = (size_t)Q * C;
  unpool_scatter_kernel<<<(unsigned)cdiv64(n, 256), 256, 0, (cudaStream_t)stream>>>(G, ldg, gp, ldp, arg, Q, C, accumulate);
  return check_launch("unpool_scatter_kernel");
}

extern "C" int usip_knn_combine_bwd(const float* GY, int ldg, const float* pts, const int32_t* knn_idx, float* GZ,
                                    int ldz, float* gW, int ldw, int B, int M, int K, int C, void* stream) {
  USIP_REQUIRE(GY && pts && knn_idx && GZ && gW && C % 4 == 0 && ldg % 4 == 0, "knn_combine_bwd: bad args");
  USIP_REQUIRE((reinterpret_cast<uintptr_t>(GY) & 15) == 0, "knn_combine_bwd: GY must be 16-byte aligned");
  int G = B * M * K;
  knn_combine_bwd_kernel<<<cdiv(G, BW_ROWS), 256, (size_t)C * 3 * sizeof(float), (cudaStream_t)stream>>>(
      GY, ldg, pts, knn_idx, GZ, ldz, gW, ldw, B, M, K, C);
  return check_launch("knn_combine_bwd_kernel");
}

extern "C" int usip_colsum(const float* G, int ldg, float* out, int P, int C, void* stream) {
  USIP_REQUIRE(G && out, "colsum: bad args");
  if (C % 4 == 0 && C <= 1024 && ldg % 4 == 0 && (reinterpret_cast<uintptr_t>(G) % 16) == 0) {
    const int rpp = 256 / (C / 4);
    const int blocks = (int)min((long long)cdiv(P, rpp * 4), (long long)device_sm_count() * 8);
    colsum_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(G, ldg, out, P, C);
    return check_launch("colsum_kernel");
  }
  dim3 grid(cdiv(P, 1024), cdiv(C, 256));
  colsum_slow_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(G, ldg, out, P, C);
  return check_launch("colsum_slow_kernel");
}

extern "C" int usip_head_bwd(const float* g_kp, const float* g_sig, const float* out4, int ld, float* G, int B, int M,
                             void* stream) {
  USIP_REQUIRE(out4 && G, "head_bwd: bad args");
  USIP_REQUIRE((reinterpret_cast<uintptr_t>(G) & 15) == 0, "head_bwd: G must be 16-byte aligned");
  head_bwd_kernel<<<cdiv(B * M, 256), 256, 0, (cudaStream_t)stream>>>(g_kp, g_sig, out4, ld, G, B, M);
  return check_launch("head_bwd_kernel");
}

namespace usip {
int wgrad_tc(const float* GY, int ldg, const float* X, int ldx, const float* sc, const float* sh, int relu, float* gW,
             int ldw, int P, int Cout, int Cin, int single, cudaStream_t st);   // wgrad_tc.cu (-2: shape not eligible)
}

extern "C" int usip_wgrad(const float* GY, int ldg, const float* X, int ldx, const float* in_scale,
                          const float* in_shift, int in_relu, float* gW, int ldw, int P, int Cout, int Cin,
                          int precision, void* stream) {
  USIP_REQUIRE(GY && X && gW && P > 0 && Cout > 0 && Cin > 0 && (!in_scale == !in_shift), "wgrad: bad args");
  if (precision == 1 || precision == 4) {            // 1: 3xTF32 (fp32-equivalent), 4: plain TF32 (one MMA per MAC)
    int rc = wgrad_tc(GY, ldg, X, ldx, in_scale, in_shift, in_relu, gW, ldw, P, Cout, Cin, precision == 4, (cudaStream_t)stream);
    if (rc != -2) return rc;
  }
  if (Cin <= 8 && (Cout == 32 || Cout == 64 || Cout == 128 || Cout == 256) && P >= 4096 && ldg % 4 == 0 &&
      (reinterpret_cast<uintptr_t>(GY) & 15) == 0) {
    const int rpp = 1024 / Cout;
    const int blocks = (int)min((long long)cdiv(P, rpp * 8), (long long)device_sm_count() * 2);      // few CTAs: each ends in Cout*Cin atomics on the same words
    wgrad_narrow_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(GY, ldg, X, ldx, in_scale, in_shift, in_relu, gW, ldw, P, Cout, Cin);
    return check_launch("wgrad_narrow_kernel");
  }
  const int tiles = cdiv(Cout, 128) * cdiv(Cin, 128);
  int splits = max(1, min(cdiv(P, 128), (device_sm_count() * 4) / tiles));
  int rows = cdiv(cdiv(P, splits), WG_BK) * WG_BK;
  splits = cdiv(P, rows);
  dim3 grid(splits, cdiv(Cout, 128), cdiv(Cin, 128));
  wgrad_simt_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(GY, ldg, X, ldx, in_scale, in_shift, in_relu, gW, ldw, P, Cout,
                                                            Cin, rows);
  return check_launch("wgrad_simt_kernel");
}

extern "C" int usip_l2norm_bwd(const float* g, const float* Y, int ldy, float* GY, int ldg, int B, int M, int C, void* stream) {
  USIP_REQUIRE(g && Y && GY && ldy >= C && ldg >= C, "l2norm_bwd: bad args");
  l2norm_bwd_kernel<<<cdiv(B * M * 32, 256), 256, 0, (cudaStream_t)stream>>>(g, Y, ldy, GY, ldg, B, M, C);
  return check_launch("l2norm_bwd_kernel");
}

extern "C" int usip_desc_triplet_bwd(const float* anc, const float* pos, const float* neg, const float* dpos,
                                     const int32_t* ipos, const float* dneg, const int32_t* ineg, const float* sigma,
                                     float gamma, float sigma_max, const float* g_loss, float* g_anc, float* g_pos,
                                     float* g_neg, int B, int C, int M, int Mp, int Mn, void* stream) {
  USIP_REQUIRE(anc && pos && neg && dpos && ipos && dneg && ineg && sigma && g_loss && g_anc && g_pos && g_neg,
               "desc_triplet_bwd: bad args");
  desc_triplet_bwd_kernel<<<dim3(M, B), 128, 0, (cudaStream_t)stream>>>(anc, pos, neg, dpos, ipos, dneg, ineg, sigma, gamma,
                                                                       sigma_max, g_loss, g_anc, g_pos, g_neg, C, M, Mp, Mn);
  return check_launch("desc_triplet_bwd_kernel");
}
