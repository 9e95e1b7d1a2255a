// mlp.cu -- shared-MLP stack building blocks (fp32 SIMT path).
//   usip_layer_fwd      : Y = act(X) W^T + bias (+ per-group addend), act = folded BatchNorm + ReLU of the
//                         PREVIOUS layer applied on operand load; epilogue emits BN statistic partials and
//                         per-group max/min (+arg) of the raw output so max_k relu(bn(y_k)) never needs a
//                         second pass (relu o affine is monotone: max if scale>=0, min otherwise).
//   usip_bn_finalize    : deterministic reduction of the partials -> folded affine + running stats
//   usip_knn_combine    : first kNN-fusion layer from a per-node GEMM result (no (B,131,M,K) tensor)
// Reference: models/layers.py:23-121 (MyBatchNorm*), :172-216 (MyConv2d), :248-303 (EquivariantLayer),
//            :401-440 (GeneralKNNFusionModule), models/networks.py:143-154 (head).
#include "common.cuh"

namespace usip {

constexpr int L_BM = 128;      // rows per CTA tile == stat tile
constexpr int L_BK = 16;
constexpr int L_THREADS = 256;
constexpr int L_LDS = L_BM + 4;

template <int BN>
struct LayerSmem {
  static constexpr int A_FLOATS = 2 * L_BK * L_LDS;
  static constexpr int B_FLOATS = 2 * L_BK * (BN + 4);
  static constexpr int MAIN_BYTES = (A_FLOATS + B_FLOATS) * 4;
  static constexpr int EPI_BYTES = 32 * BN * 8;            // chunk value + chunk arg
  static constexpr int RED_BYTES = 2 * 16 * BN * 4;        // stat reduction
  static constexpr int BYTES = MAIN_BYTES > EPI_BYTES ? (MAIN_BYTES > RED_BYTES ? MAIN_BYTES : RED_BYTES)
                                                      : (EPI_BYTES > RED_BYTES ? EPI_BYTES : RED_BYTES);
};

template <int BN>
__global__ void __launch_bounds__(L_THREADS, 2)
layer_fwd_simt_kernel(const usip_layer_desc d) {
  constexpr int TN = BN / 16;            // 8 or 4 columns per thread
  constexpr int NH = TN / 4;             // column halves (2 or 1)
  constexpr int LDB = BN + 4;
  extern __shared__ __align__(16) float smem[];
  float* As = smem;                                        // [2][L_BK][L_LDS]
  float* Bs = smem + LayerSmem<BN>::A_FLOATS;              // [2][L_BK][LDB]

  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  const int tile = blockIdx.x;
  const int row0 = tile * L_BM;
  const int n0 = blockIdx.y * BN;
  const int P = d.P, Cin = d.Cin, Cout = d.Cout;
  const int KT = (Cin + L_BK - 1) / L_BK;

  // ---- global -> register staging maps
  const int a_r = tid & 127, a_kh = tid >> 7;              // 8 consecutive k per thread
  const bool a_row_ok = (row0 + a_r) < P;
  const float* a_ptr = d.X + (size_t)(row0 + a_r) * d.ldx;
  const bool a_vec = ((d.ldx & 3) == 0) && ((reinterpret_cast<uintptr_t>(d.X) & 15) == 0);
  constexpr int BKH = (L_THREADS / BN);                    // k-slices for the weight tile: 2 (BN=128) / 4 (BN=64)
  constexpr int BKW = L_BK / BKH;                          // k per thread: 8 / 4
  const int b_n = tid % BN, b_kh = tid / BN;
  const bool b_row_ok = (n0 + b_n) < Cout;
  const float* b_ptr = d.w_transposed ? d.W + (n0 + b_n) : d.W + (size_t)(n0 + b_n) * d.ldw;
  const bool b_vec = !d.w_transposed && ((d.ldw & 3) == 0) && ((reinterpret_cast<uintptr_t>(d.W) & 15) == 0);
  const bool has_affine = d.in_scale != nullptr;

  float a_reg[8], b_reg[BKW];

  auto load_tile = [&](int kt) {
    const int k0 = kt * L_BK + a_kh * 8;
    if (a_row_ok && a_vec && k0 + 8 <= Cin) {
      float4 v0 = *reinterpret_cast<const float4*>(a_ptr + k0);
      float4 v1 = *reinterpret_cast<const float4*>(a_ptr + k0 + 4);
      a_reg[0] = v0.x; a_reg[1] = v0.y; a_reg[2] = v0.z; a_reg[3] = v0.w;
      a_reg[4] = v1.x; a_reg[5] = v1.y; a_reg[6] = v1.z; a_reg[7] = v1.w;
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) a_reg[j] = (a_row_ok && k0 + j < Cin) ? a_ptr[k0 + j] : 0.f;
    }
    if (has_affine) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        int k = k0 + j;
        if (k < Cin) {
          float v = fmaf(a_reg[j], __ldg(d.in_scale + k), __ldg(d.in_shift + k));
          a_reg[j] = d.in_relu ? fmaxf(v, 0.f) : v;
        }
      }
    } else if (d.in_relu) {
#pragma unroll
      for (int j = 0; j < 8; ++j) a_reg[j] = fmaxf(a_reg[j], 0.f);
    }
    const int kb = kt * L_BK + b_kh * BKW;
    if (b_row_ok && b_vec && kb + BKW <= Cin) {
#pragma unroll
      for (int j = 0; j < BKW; j += 4) {
        float4 v = *reinterpret_cast<const float4*>(b_ptr + kb + j);
        b_reg[j] = v.x; b_reg[j + 1] = v.y; b_reg[j + 2] = v.z; b_reg[j + 3] = v.w;
      }
    } else {
#pragma unroll
      for (int j = 0; j < BKW; ++j)
        b_reg[j] = (b_row_ok && kb + j < Cin) ? (d.w_transposed ? b_ptr[(size_t)(kb + j) * d.ldw] : b_ptr[kb + j]) : 0.f;
    }
  };
  auto store_tile = [&](int buf) {
    float* A = As + buf * L_BK * L_LDS;
    float* Bm = Bs + buf * L_BK * LDB;
#pragma unroll
    for (int j = 0; j < 8; ++j) A[(a_kh * 8 + j) * L_LDS + a_r] = a_reg[j];
#pragma unroll
    for (int j = 0; j < BKW; ++j) Bm[(b_kh * BKW + j) * LDB + b_n] = b_reg[j];
  };

  float acc[8][TN];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

  load_tile(0);
  store_tile(0);
  __syncthreads();
  for (int kt = 0; kt < KT; ++kt) {
    const int buf = kt & 1;
    if (kt + 1 < KT) load_tile(kt + 1);
    const float* A = As + buf * L_BK * L_LDS;
    const float* Bm = Bs + buf * L_BK * LDB;
#pragma unroll
    for (int k = 0; k < L_BK; ++k) {
      float a[8], b[TN];
      float4 a0 = *reinterpret_cast<const float4*>(A + k * L_LDS + ty * 4);
      float4 a1 = *reinterpret_cast<const float4*>(A + k * L_LDS + 64 + ty * 4);
      a[0] = a0.x; a[1] = a0.y; a[2] = a0.z; a[3] = a0.w; a[4] = a1.x; a[5] = a1.y; a[6] = a1.z; a[7] = a1.w;
#pragma unroll
      for (int h = 0; h < NH; ++h) {
        float4 bv = *reinterpret_cast<const float4*>(Bm + k * LDB + h * 64 + tx * 4);
        b[h * 4 + 0] = bv.x; b[h * 4 + 1] = bv.y; b[h * 4 + 2] = bv.z; b[h * 4 + 3] = bv.w;
      }
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    if (kt + 1 < KT) store_tile(buf ^ 1);
    __syncthreads();
  }

  // ---- epilogue: thread rows r(i) = (i<4 ? ty*4+i : 64+ty*4+i-4), cols c(j) = (j/4)*64 + tx*4 + j%4
  int rows[8]; bool rok[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) { rows[i] = row0 + (i < 4 ? ty * 4 + i : 64 + ty * 4 + (i - 4)); rok[i] = rows[i] < P; }
  int cols[TN]; bool cok[TN];
#pragma unroll
  for (int j = 0; j < TN; ++j) { cols[j] = n0 + (j >> 2) * 64 + tx * 4 + (j & 3); cok[j] = cols[j] < Cout; }

  if (d.bias) {
#pragma unroll
    for (int j = 0; j < TN; ++j) {
      float bv = cok[j] ? __ldg(d.bias + cols[j]) : 0.f;
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[i][j] += bv;
    }
  }
  if (d.addend) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      if (!rok[i]) continue;
      int g = d.add_index ? __ldg(d.add_index + rows[i]) : rows[i] / d.add_group;
      const float* ap = d.addend + (size_t)g * d.ld_add;
#pragma unroll
      for (int j = 0; j < TN; ++j) if (cok[j]) acc[i][j] += __ldg(ap + cols[j]);
    }
  }
  if (d.Y) {
    const bool y_vec = ((d.ldy & 3) == 0) && ((reinterpret_cast<uintptr_t>(d.Y) & 15) == 0) && (Cout % 4 == 0);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      if (!rok[i]) continue;
      float* yp = d.Y + (size_t)rows[i] * d.ldy;
#pragma unroll
      for (int h = 0; h < NH; ++h) {
        if (y_vec && cok[h * 4]) {
          *reinterpret_cast<float4*>(yp + cols[h * 4]) =
              make_float4(acc[i][h * 4], acc[i][h * 4 + 1], acc[i][h * 4 + 2], acc[i][h * 4 + 3]);
        } else {
#pragma unroll
          for (int j = 0; j < 4; ++j) if (cok[h * 4 + j]) yp[cols[h * 4 + j]] = acc[i][h * 4 + j];
        }
      }
    }
  }

  // ---- BN statistic partials: reduce the 16 row-owners of each column in fixed order
  if (d.stat_partial) {
    float* red = smem;                                       // [2][16][BN]
#pragma unroll
    for (int j = 0; j < TN; ++j) {
      float s = 0.f, ss = 0.f;
#pragma unroll
      for (int i = 0; i < 8; ++i) if (rok[i]) { s += acc[i][j]; ss = fmaf(acc[i][j], acc[i][j], ss); }
      int cl = (j >> 2) * 64 + tx * 4 + (j & 3);
      red[ty * BN + cl] = s;
      red[16 * BN + ty * BN + cl] = ss;
    }
    __syncthreads();
    if (tid < BN && n0 + tid < Cout) {
      float s = 0.f, ss = 0.f;
#pragma unroll
      for (int t = 0; t < 16; ++t) { s += red[t * BN + tid]; ss += red[16 * BN + t * BN + tid]; }
      d.stat_partial[((size_t)tile * 2 + 0) * Cout + n0 + tid] = s;
      d.stat_partial[((size_t)tile * 2 + 1) * Cout + n0 + tid] = ss;
    }
    __syncthreads();
  }

  // ---- per-group max / min (+ row-in-group arg).  chunk = 4 consecutive rows owned by one thread.
  if (d.gmax || d.gmin) {
    float* cval = smem;                                      // [32][BN]
    int* carg = reinterpret_cast<int*>(smem + 32 * BN);      // [32][BN]
    const int g = d.group, cpg = g >> 2, groups_per_tile = L_BM / g;
    for (int pass = 0; pass < 2; ++pass) {
      float* gout = pass == 0 ? d.gmax : d.gmin;
      int32_t* aout = pass == 0 ? d.garg_max : d.garg_min;
      if (!gout) continue;
#pragma unroll
      for (int j = 0; j < TN; ++j) {
        int cl = (j >> 2) * 64 + tx * 4 + (j & 3);
#pragma unroll
        for (int hrow = 0; hrow < 2; ++hrow) {
          float best = pass == 0 ? -INFINITY : INFINITY; int bi = 0;
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            float v = acc[hrow * 4 + i][j];
            bool better = rok[hrow * 4 + i] && (pass == 0 ? v > best : v < best);
            if (better) { best = v; bi = i; }
          }
          int chunk = hrow * 16 + ty;                        // rows chunk*4 .. chunk*4+3 of the tile
          cval[chunk * BN + cl] = best; carg[chunk * BN + cl] = chunk * 4 + bi;
        }
      }
      __syncthreads();
      for (int t = tid; t < groups_per_tile * BN; t += L_THREADS) {
        int gi = t / BN, cl = t - gi * BN;
        int grow = (row0 / g) + gi;
        if (n0 + cl < Cout && (size_t)grow * g < (size_t)P) {
          float best = pass == 0 ? -INFINITY : INFINITY; int bi = gi * g;
          for (int c = 0; c < cpg; ++c) {
            float v = cval[(gi * cpg + c) * BN + cl];
            bool better = pass == 0 ? v > best : v < best;
            if (better) { best = v; bi = carg[(gi * cpg + c) * BN + cl]; }
          }
          gout[(size_t)grow * Cout + n0 + cl] = best;
          if (aout) aout[(size_t)grow * Cout + n0 + cl] = bi - gi * g;
        }
      }
      __syncthreads();
    }
  }
}

// ------------------------------------------------------------------------------------------------
constexpr int BNF_C = 8;       // channels per CTA: one 32-byte sector per partial row, C/8 CTAs
constexpr int BNF_T = 256;     // threads: 8 channels x 32 partial-row slices
__global__ void __launch_bounds__(BNF_T)
bn_finalize_kernel(const float* __restrict__ part, int ntiles, double count, int C,
                   const float* __restrict__ gamma, const float* __restrict__ beta, float eps, float momentum,
                   float* __restrict__ running_mean, float* __restrict__ running_var,
                   float* __restrict__ scale, float* __restrict__ shift,
                   float* __restrict__ save_mean, float* __restrict__ save_invstd) {
  // block = 8 channels x 32 partial-row slices; every thread keeps 8 independent loads in flight per batch; the slices
  // meet by two warp shuffles and ONE barrier (round 1: 1024 threads and a seven-level shared-memory tree of doubles --
  // 8 us per launch, ten launches per forward step).  Fixed order -> deterministic.
  constexpr int SL = BNF_T / BNF_C;
  __shared__ double sh[2][BNF_T / 32][BNF_C];
  const int cl = threadIdx.x % BNF_C, sl = threadIdx.x / BNF_C;
  const int c = blockIdx.x * BNF_C + cl;
  double s = 0.0, ss = 0.0;
  if (c < C) {
    int t = sl;
    for (; t + 7 * SL < ntiles; t += 8 * SL) {
      float a[8], b[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        a[u] = __ldg(part + ((size_t)(t + u * SL) * 2 + 0) * C + c);
        b[u] = __ldg(part + ((size_t)(t + u * SL) * 2 + 1) * C + c);
      }
#pragma unroll
      for (int u = 0; u < 8; ++u) { s += (double)a[u]; ss += (double)b[u]; }
    }
    if (t < ntiles) {                                          // tail batch: clamped addresses, no branch around the loads
      float a[8], b[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const int tt = min(t + u * SL, ntiles - 1);
        a[u] = __ldg(part + ((size_t)tt * 2 + 0) * C + c);
        b[u] = __ldg(part + ((size_t)tt * 2 + 1) * C + c);
      }
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const bool ok = t + u * SL < ntiles;
        s += ok ? (double)a[u] : 0.0; ss += ok ? (double)b[u] : 0.0;
      }
    }
  }
  // a warp holds 4 slices x 8 channels (lane = 8*slice + channel): fold the slices, then the 8 warps
  s += __shfl_xor_sync(0xffffffffu, s, 8); ss += __shfl_xor_sync(0xffffffffu, ss, 8);
  s += __shfl_xor_sync(0xffffffffu, s, 16); ss += __shfl_xor_sync(0xffffffffu, ss, 16);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane < BNF_C) { sh[0][warp][lane] = s; sh[1][warp][lane] = ss; }
  __syncthreads();
  if (sl == 0 && c < C) {
    double S = 0.0, SS = 0.0;
#pragma unroll
    for (int w2 = 0; w2 < BNF_T / 32; ++w2) { S += sh[0][w2][cl]; SS += sh[1][w2][cl]; }
    double mean = S / count;
    double var = SS / count - mean * mean;
    if (var < 0.0) var = 0.0;
    double invstd = 1.0 / sqrt(var + (double)eps);
    float g = gamma ? gamma[c] : 1.f, b = beta ? beta[c] : 0.f;
    float sc = (float)((double)g * invstd);
    scale[c] = sc;
    shift[c] = (float)((double)b - mean * (double)g * invstd);
    if (save_mean) save_mean[c] = (float)mean;
    if (save_invstd) save_invstd[c] = (float)invstd;
    if (running_mean) running_mean[c] = (float)((1.0 - momentum) * running_mean[c] + momentum * mean);
    if (running_var) {
      double unb = count > 1.0 ? var * count / (count - 1.0) : var;
      running_var[c] = (float)((1.0 - momentum) * running_var[c] + momentum * unb);
    }
  }
}

__global__ void bn_eval_affine_kernel(const float* __restrict__ gamma, const float* __restrict__ beta,
                                      const float* __restrict__ rm, const float* __restrict__ rv, float eps, int C,
                                      float* __restrict__ scale, float* __restrict__ shift) {
  int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  float invstd = 1.0f / sqrtf(rv[c] + eps);
  float sc = gamma[c] * invstd;
  scale[c] = sc; shift[c] = beta[c] - rm[c] * sc;
}

// ------------------------------------------------------------------------------------------------
// knn_combine: rows (b,m,k); warp w owns rows w, w+8, ... of the 128-row tile; lanes own float4 channel
// groups.  Y = Z[neighbour] + Wxyz*(p_nb - p_m) + bias, plus BN stat partials.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
knn_combine_kernel(const float* __restrict__ Z, int ldz, const float* __restrict__ pts,
                   const int32_t* __restrict__ knn_idx, const float* __restrict__ W, int ldw,
                   const float* __restrict__ bias, float* __restrict__ Y, int ldy, float* __restrict__ part,
                   int B, int M, int K, int Cout) {
  extern __shared__ float red[];                             // [2][8][Cout]
  const int tile = blockIdx.x, row0 = tile * L_BM;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int G = B * M * K;
  // the neighbour offsets of the warp's rows (row0 + warp + 8 i, i < 16) are computed ONCE, by lane i, and broadcast by
  // shuffles inside the channel loop -- every lane used to redo the two integer divisions, the index load and the six
  // coordinate loads for every row and every 128-channel pass
  static_assert(L_BM / 8 <= 32, "one lane per row of the warp");
  int nb_row = 0; float ndx = 0.f, ndy = 0.f, ndz = 0.f;
  {
    const int r = row0 + warp + 8 * lane;
    if (lane < L_BM / 8 && r < G) {
      const int q = r / K;                                   // global node id b*M+m
      const int b = q / M, m = q - b * M;
      const int j = knn_idx[r];
      const float* p = pts + (size_t)b * 3 * M;
      ndx = p[j] - p[m]; ndy = p[M + j] - p[M + m]; ndz = p[2 * M + j] - p[2 * M + m];            // layers.py:428
      nb_row = b * M + j;
    }
  }
  for (int c4 = lane; c4 * 4 < ((Cout + 127) / 128) * 128; c4 += 32) {       // uniform trip count: the shuffles need every lane
    const bool act = c4 * 4 < Cout;
    float w0[4], w1[4], w2[4], bs[4], s[4] = {0, 0, 0, 0}, ss[4] = {0, 0, 0, 0};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float* wr = W + (size_t)(act ? c4 * 4 + j : 0) * ldw;
      w0[j] = wr[0]; w1[j] = wr[1]; w2[j] = wr[2]; bs[j] = (bias && act) ? bias[c4 * 4 + j] : 0.f;
    }
    int i = 0;
    for (int r = row0 + warp; r < min(row0 + L_BM, G); r += 8, ++i) {
      const int zr = __shfl_sync(0xffffffffu, nb_row, i);
      const float dx = __shfl_sync(0xffffffffu, ndx, i), dy = __shfl_sync(0xffffffffu, ndy, i), dz = __shfl_sync(0xffffffffu, ndz, i);
      if (act) {
        float4 z = *reinterpret_cast<const float4*>(Z + (size_t)zr * ldz + c4 * 4);
        float y[4] = {z.x, z.y, z.z, z.w};
#pragma unroll
        for (int t = 0; t < 4; ++t) {
          y[t] += fmaf(w2[t], dz, fmaf(w1[t], dy, w0[t] * dx)) + bs[t];
          s[t] += y[t]; ss[t] = fmaf(y[t], y[t], ss[t]);
        }
        *reinterpret_cast<float4*>(Y + (size_t)r * ldy + c4 * 4) = make_float4(y[0], y[1], y[2], y[3]);
      }
    }
    if (act) {
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        red[(0 * 8 + warp) * Cout + c4 * 4 + t] = s[t];
        red[(1 * 8 + warp) * Cout + c4 * 4 + t] = ss[t];
      }
    }
  }
  __syncthreads();
  if (part)
    for (int c = threadIdx.x; c < Cout; c += 256) {
      float s = 0.f, ss = 0.f;
#pragma unroll
      for (int w = 0; w < 8; ++w) { s += red[(0 * 8 + w) * Cout + c]; ss += red[(1 * 8 + w) * Cout + c]; }
      part[((size_t)tile * 2 + 0) * Cout + c] = s;
      part[((size_t)tile * 2 + 1) * Cout + c] = ss;
    }
}

__global__ void group_select_kernel(const float* __restrict__ gmax, const float* __restrict__ gmin,
                                    const float* __restrict__ scale, const float* __restrict__ shift,
                                    float* __restrict__ out, int ldo, int Q, int C) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)Q * C) return;
  int q = (int)(i / C), c = (int)(i - (size_t)q * C);
  float sc = scale[c];
  float v = sc >= 0.f ? gmax[i] : gmin[i];
  out[(size_t)q * ldo + c] = fmaxf(fmaf(v, sc, shift[c]), 0.f);
}

// four channels per thread (C % 4 == 0, 16-byte aligned rows): three 16-byte loads and one 16-byte store per thread
__global__ void group_select4_kernel(const float* __restrict__ gmax, const float* __restrict__ gmin,
                                     const float* __restrict__ scale, const float* __restrict__ shift,
                                     float* __restrict__ out, int ldo, int Q, int C) {
  const int c4n = C >> 2;
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)Q * c4n) return;
  const int q = (int)(i / c4n), c = (int)(i - (size_t)q * c4n) * 4;
  const float4 sc = __ldg(reinterpret_cast<const float4*>(scale + c)), sh = __ldg(reinterpret_cast<const float4*>(shift + c));
  const float4 hi = __ldg(reinterpret_cast<const float4*>(gmax + (size_t)q * C + c));
  const float4 lo = __ldg(reinterpret_cast<const float4*>(gmin + (size_t)q * C + c));
  float4 o;
  o.x = fmaxf(fmaf(sc.x >= 0.f ? hi.x : lo.x, sc.x, sh.x), 0.f);
  o.y = fmaxf(fmaf(sc.y >= 0.f ? hi.y : lo.y, sc.y, sh.y), 0.f);
  o.z = fmaxf(fmaf(sc.z >= 0.f ? hi.z : lo.z, sc.z, sh.z), 0.f);
  o.w = fmaxf(fmaf(sc.w >= 0.f ? hi.w : lo.w, sc.w, sh.w), 0.f);
  *reinterpret_cast<float4*>(out + (size_t)q * ldo + c) = o;
}

__global__ void head_finalize_kernel(const float* __restrict__ out4, int ld, const float* __restrict__ cmean,
                                     float lb, float* __restrict__ kp, float* __restrict__ sig, int B, int M) {
  int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= B * M) return;
  int b = t / M, m = t - b * M;
  const float* o = out4 + (size_t)t * ld;
#pragma unroll
  for (int c = 0; c < 3; ++c)
    kp[(size_t)b * 3 * M + (size_t)c * M + m] = o[c] + cmean[(size_t)b * 3 * M + (size_t)c * M + m];   // networks.py:151
  float x = o[3];
  sig[t] = (x > 20.f ? x : log1pf(expf(x))) + lb;                                                     // networks.py:72,154
}

// Narrow output layers (Cout <= 8, e.g. the 256->4 head): one warp per row, lanes stride over K, weights in shared
// memory, warp-shuffle reduction.  Same prologue as the tiled kernels; no statistics / group epilogue.
template <int NOUT>
__global__ void __launch_bounds__(256)
layer_fwd_rowwarp_kernel(const usip_layer_desc d) {
  extern __shared__ float sw[];                         // [NOUT][Cin] weights, then scale/shift [2][Cin]
  const int Cin = d.Cin, Cout = d.Cout;
  for (int i = threadIdx.x; i < NOUT * Cin; i += 256) {
    const int n = i / Cin, k = i - n * Cin;
    sw[i] = n < Cout ? (d.w_transposed ? d.W[(size_t)k * d.ldw + n] : d.W[(size_t)n * d.ldw + k]) : 0.f;
  }
  float* ssc = sw + NOUT * Cin; float* ssh = ssc + Cin;
  for (int k = threadIdx.x; k < Cin; k += 256) { ssc[k] = d.in_scale ? d.in_scale[k] : 1.f; ssh[k] = d.in_shift ? d.in_shift[k] : 0.f; }
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (row >= d.P) return;
  const float* x = d.X + (size_t)row * d.ldx;
  float acc[NOUT];
#pragma unroll
  for (int n = 0; n < NOUT; ++n) acc[n] = 0.f;
  for (int k = lane; k < Cin; k += 32) {
    float a = fmaf(x[k], ssc[k], ssh[k]);
    if (d.in_relu) a = fmaxf(a, 0.f);
#pragma unroll
    for (int n = 0; n < NOUT; ++n) acc[n] = fmaf(a, sw[n * Cin + k], acc[n]);
  }
#pragma unroll
  for (int n = 0; n < NOUT; ++n) acc[n] = warp_sum(acc[n]);
  if (lane < Cout && lane < NOUT) {
    float v = 0.f;
#pragma unroll
    for (int n = 0; n < NOUT; ++n) if (lane == n) v = acc[n];
    if (d.bias) v += d.bias[lane];
    if (d.Y) d.Y[(size_t)row * d.ldy + lane] = v;
  }
}

// First layer of a point stack: Cin <= 8 input channels (xyz + surface normal), Cout in {32, 64}, raw input (no folded
// BN), Y + BN statistics out.  HBM-bound (8 B in, 4*Cout B out per row); the generic 128x64x16 register tile pads K to
// 16 and ran at 25 % of that roofline.  CTA = 128 rows, 4 warps x 32 rows; a lane owns channels lane (and lane + 32)
// with their <= 8 weights in registers, so a row costs two broadcast shared loads, <= 16 FMAs and one / two coalesced
// 128-byte stores.  One statistics partial per CTA = per 128-row tile, like the generic SIMT kernel.
template <int NCH>                                   // channels per lane: Cout = 32 * NCH
__global__ void __launch_bounds__(128)
layer_fwd_narrow_kernel(const usip_layer_desc d) {
  __shared__ float4 sx[128][2];
  __shared__ float sred[4][2][32 * NCH];
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  const int row0 = blockIdx.x * 128;
  const int P = d.P, Cin = d.Cin, Cout = d.Cout;
  {   // stage the 128 x 8 input tile (zero padded)
    const int r = row0 + tid;
    float v[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    if (r < P) {
      const float* x = d.X + (size_t)r * d.ldx;
      if (d.ldx >= 8 && (d.ldx & 3) == 0 && (reinterpret_cast<uintptr_t>(d.X) & 15) == 0) {
        const float4 a = *reinterpret_cast<const float4*>(x), b = *reinterpret_cast<const float4*>(x + 4);
        v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
        for (int k = Cin; k < 8; ++k) v[k] = 0.f;
      } else {
        for (int k = 0; k < Cin; ++k) v[k] = x[k];
      }
    }
    sx[tid][0] = make_float4(v[0], v[1], v[2], v[3]); sx[tid][1] = make_float4(v[4], v[5], v[6], v[7]);
  }
  float wr[NCH][8], br[NCH];
#pragma unroll
  for (int c = 0; c < NCH; ++c) {
    const int n = lane + 32 * c;
#pragma unroll
    for (int k = 0; k < 8; ++k) wr[c][k] = k < Cin ? (d.w_transposed ? d.W[(size_t)k * d.ldw + n] : d.W[(size_t)n * d.ldw + k]) : 0.f;
    br[c] = d.bias ? d.bias[n] : 0.f;
  }
  __syncthreads();
  float s[NCH], q[NCH];
#pragma unroll
  for (int c = 0; c < NCH; ++c) { s[c] = 0.f; q[c] = 0.f; }
  const int nrows = min(32, max(0, P - (row0 + w * 32)));
  for (int r = 0; r < nrows; ++r) {
    const float4 a = sx[w * 32 + r][0], b = sx[w * 32 + r][1];
    const size_t row = (size_t)row0 + w * 32 + r;
#pragma unroll
    for (int c = 0; c < NCH; ++c) {
      float y = br[c];
      y = fmaf(a.x, wr[c][0], y); y = fmaf(a.y, wr[c][1], y); y = fmaf(a.z, wr[c][2], y); y = fmaf(a.w, wr[c][3], y);
      y = fmaf(b.x, wr[c][4], y); y = fmaf(b.y, wr[c][5], y); y = fmaf(b.z, wr[c][6], y); y = fmaf(b.w, wr[c][7], y);
      if (d.Y) d.Y[row * d.ldy + lane + 32 * c] = y;
      s[c] += y; q[c] = fmaf(y, y, q[c]);
    }
  }
  if (d.stat_partial) {
#pragma unroll
    for (int c = 0; c < NCH; ++c) { sred[w][0][lane + 32 * c] = s[c]; sred[w][1][lane + 32 * c] = q[c]; }
    __syncthreads();
    for (int i = tid; i < 2 * Cout; i += 128) {
      const int which = i / Cout, n = i - which * Cout;
      d.stat_partial[((size_t)blockIdx.x * 2 + which) * Cout + n] =
          (sred[0][which][n] + sred[1][which][n]) + (sred[2][which][n] + sred[3][which][n]);
    }
  }
}

// descriptor / (||descriptor||_2 + 1e-5) over channels, [Q,C] rows -> reference (B,C,M) layout (networks.py:383)
__global__ void __launch_bounds__(256)
l2norm_to_bcm_kernel(const float* __restrict__ X, int ldx, float* __restrict__ out, float* __restrict__ norm_out, int B,
                     int M, int C) {
  const int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (w >= B * M) return;
  const int b = w / M, m = w - b * M;
  const float* x = X + (size_t)w * ldx;
  float ss = 0.f;
  for (int c = lane; c < C; c += 32) ss = fmaf(x[c], x[c], ss);
  ss = warp_sum(ss);
  const float nrm = sqrtf(ss);
  const float inv = 1.0f / (nrm + 1e-5f);
  if (norm_out && lane == 0) norm_out[w] = nrm;
  for (int c = lane; c < C; c += 32) out[((size_t)b * C + c) * M + m] = x[c] * inv;
}

template <int BN>
static int launch_layer_simt(const usip_layer_desc& d, cudaStream_t st) {
  static bool attr_done = false;
  if (!attr_done) {
    cudaError_t e = cudaFuncSetAttribute(layer_fwd_simt_kernel<BN>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         LayerSmem<BN>::BYTES);
    if (e != cudaSuccess) { set_last_error("layer_fwd smem attr"); return (int)e; }
    attr_done = true;
  }
  dim3 grid(cdiv(d.P, L_BM), cdiv(d.Cout, BN));
  layer_fwd_simt_kernel<BN><<<grid, L_THREADS, LayerSmem<BN>::BYTES, st>>>(d);
  return check_launch("layer_fwd_simt_kernel");
}

int layer_fwd_tc(const usip_layer_desc& d, cudaStream_t st);   // mlp_tc.cu
int tc_stat_slots(const usip_layer_desc& d);
int tc_pack_many(const usip_layer_desc* descs, int n, cudaStream_t st);

}  // namespace usip

using namespace usip;

extern "C" int usip_layer_tile_rows(void) { return L_BM; }
extern "C" int usip_layer_stat_slots(const usip_layer_desc* dp) {
  if (!dp || dp->P <= 0 || dp->Cout <= 0) return 0;
  return dp->precision != 0 ? tc_stat_slots(*dp) : cdiv(dp->P, L_BM);
}
extern "C" int64_t usip_layer_tc_workspace_bytes(int Cin, int Cout) { return (int64_t)2 * Cin * Cout * 4; }

extern "C" int usip_layer_tc_pack_many(const usip_layer_desc* descs, int n, void* stream) {
  USIP_REQUIRE(descs && n > 0, "layer_tc_pack_many: bad args");
  for (int i = 0; i < n; ++i) USIP_REQUIRE(descs[i].precision != 0, "layer_tc_pack_many: descriptor is not a tensor-core layer");
  return tc_pack_many(descs, n, (cudaStream_t)stream);
}

extern "C" int usip_layer_fwd(const usip_layer_desc* dp, void* stream) {
  USIP_REQUIRE(dp, "layer_fwd: null desc");
  const usip_layer_desc& d = *dp;
  USIP_REQUIRE(d.X && d.W && d.P > 0 && d.Cin > 0 && d.Cout > 0 && d.ldx >= d.Cin &&
               d.ldw >= (d.w_transposed ? d.Cout : d.Cin), "layer_fwd: bad args");
  USIP_REQUIRE(!d.Y || d.ldy >= d.Cout, "layer_fwd: bad ldy");
  USIP_REQUIRE(!d.in_scale == !d.in_shift, "layer_fwd: in_scale/in_shift must come together");
  if (d.gmax || d.gmin) {
    USIP_REQUIRE(d.group >= 4 && (d.group % 4) == 0 && (L_BM % d.group) == 0 && (d.P % d.group) == 0,
                 "layer_fwd: group must divide 128 and P and be a multiple of 4");
  }
  if (d.addend) USIP_REQUIRE(d.add_index || d.add_group > 0, "layer_fwd: addend needs add_index or add_group");
  cudaStream_t st = (cudaStream_t)stream;
  if (d.precision == 1) return layer_fwd_tc(d, st);
  if (d.Cout <= 8 && !d.stat_partial && !d.gmax && !d.gmin && !d.addend && (size_t)(8 + 2) * d.Cin * 4 <= 48 * 1024) {
    const size_t smem = (size_t)(8 + 2) * d.Cin * sizeof(float);
    layer_fwd_rowwarp_kernel<8><<<cdiv(d.P, 8), 256, smem, st>>>(d);
    return check_launch("layer_fwd_rowwarp_kernel");
  }
  if (d.Cin <= 8 && (d.Cout == 32 || d.Cout == 64) && !d.in_scale && !d.in_relu && !d.addend && !d.gmax && !d.gmin) {
    if (d.Cout == 64) layer_fwd_narrow_kernel<2><<<cdiv(d.P, 128), 128, 0, st>>>(d);
    else layer_fwd_narrow_kernel<1><<<cdiv(d.P, 128), 128, 0, st>>>(d);
    return check_launch("layer_fwd_narrow_kernel");
  }
  if (d.Cout <= 64) return launch_layer_simt<64>(d, st);
  return launch_layer_simt<128>(d, st);
}

extern "C" int usip_bn_finalize(const float* stat_partial, int ntiles, int64_t count, int C, const float* gamma,
                                const float* beta, float eps, float momentum, float* running_mean,
                                float* running_var, float* scale, float* shift, float* save_mean,
                                float* save_invstd, void* stream) {
  USIP_REQUIRE(stat_partial && scale && shift && ntiles > 0 && count > 0 && C > 0, "bn_finalize: bad args");
  bn_finalize_kernel<<<cdiv(C, BNF_C), BNF_T, 0, (cudaStream_t)stream>>>(stat_partial, ntiles, (double)count, C, gamma,
                                                                    beta, eps, momentum, running_mean, running_var,
                                                                    scale, shift, save_mean, save_invstd);
  return check_launch("bn_finalize_kernel");
}

extern "C" int usip_bn_eval_affine(const float* gamma, const float* beta, const float* running_mean,
                                   const float* running_var, float eps, int C, float* scale, float* shift,
                                   void* stream) {
  USIP_REQUIRE(gamma && beta && running_mean && running_var && scale && shift, "bn_eval_affine: bad args");
  bn_eval_affine_kernel<<<cdiv(C, 128), 128, 0, (cudaStream_t)stream>>>(gamma, beta, running_mean, running_var, eps,
                                                                       C, scale, shift);
  return check_launch("bn_eval_affine_kernel");
}

extern "C" int usip_knn_combine(const float* Z, int ldz, const float* pts, const int32_t* knn_idx, const float* W,
                                int ldw, const float* bias, float* Y, int ldy, float* stat_partial, int B, int M,
                                int K, int Cout, void* stream) {
  USIP_REQUIRE(Z && pts && knn_idx && W && Y && Cout % 4 == 0 && ldz % 4 == 0 && ldy % 4 == 0, "knn_combine: bad args");
  // the kernel reads Z and writes Y as float4
  USIP_REQUIRE(((reinterpret_cast<uintptr_t>(Z) | reinterpret_cast<uintptr_t>(Y)) & 15) == 0,
               "knn_combine: Z and Y must be 16-byte aligned");
  size_t smem = (size_t)2 * 8 * Cout * sizeof(float);
  USIP_REQUIRE(smem <= 48 * 1024, "knn_combine: Cout too large");
  int G = B * M * K;
  knn_combine_kernel<<<cdiv(G, L_BM), 256, smem, (cudaStream_t)stream>>>(Z, ldz, pts, knn_idx, W, ldw, bias, Y, ldy,
                                                                        stat_partial, B, M, K, Cout);
  return check_launch("knn_combine_kernel");
}

extern "C" int usip_group_select(const float* gmax, const float* gmin, const float* scale, const float* shift,
                                 float* out, int ldo, int Q, int C, void* stream) {
  USIP_REQUIRE(gmax && gmin && scale && shift && out && ldo >= C, "group_select: bad args");
  size_t n = (size_t)Q * C;
  const uintptr_t al = reinterpret_cast<uintptr_t>(gmax) | reinterpret_cast<uintptr_t>(gmin) | reinterpret_cast<uintptr_t>(scale) |
                       reinterpret_cast<uintptr_t>(shift) | reinterpret_cast<uintptr_t>(out);
  if (C % 4 == 0 && ldo % 4 == 0 && (al & 15) == 0) {
    group_select4_kernel<<<(unsigned)cdiv64(n / 4, 256), 256, 0, (cudaStream_t)stream>>>(gmax, gmin, scale, shift, out, ldo, Q, C);
    return check_launch("group_select4_kernel");
  }
  group_select_kernel<<<(unsigned)cdiv64(n, 256), 256, 0, (cudaStream_t)stream>>>(gmax, gmin, scale, shift, out, ldo, Q, C);
  return check_launch("group_select_kernel");
}

extern "C" int usip_head_finalize(const float* out4, int ld, const float* cluster_mean, float sigma_lower_bound,
                                  float* keypoints, float* sigmas, int B, int M, void* stream) {
  USIP_REQUIRE(out4 && cluster_mean && keypoints && sigmas && ld >= 4, "head_finalize: bad args");
  head_finalize_kernel<<<cdiv(B * M, 256), 256, 0, (cudaStream_t)stream>>>(out4, ld, cluster_mean, sigma_lower_bound,
                                                                          keypoints, sigmas, B, M);
  return check_launch("head_finalize_kernel");
}

extern "C" int usip_l2norm_to_bcm(const float* X, int ldx, float* out, float* norm_out, int B, int M, int C,
                                  void* stream) {
  USIP_REQUIRE(X && out && ldx >= C, "l2norm_to_bcm: bad args");
  l2norm_to_bcm_kernel<<<cdiv(B * M * 32, 256), 256, 0, (cudaStream_t)stream>>>(X, ldx, out, norm_out, B, M, C);
  return check_launch("l2norm_to_bcm_kernel");
}
