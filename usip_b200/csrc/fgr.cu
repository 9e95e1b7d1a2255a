// fgr.cu -- Fast Global Registration (Zhou, Park and Koltun, ECCV 2016) as evaluation/matlab/eval_indoor/fgr/'s mex
// runs it (LoadFeature x2, NormalizePoints, AdvancedMatching, OptimizePairwise(true, 640), GetOutputTrans), for every
// pair and every K of a keypoint-count sweep in one launch, on the mutual matches of usip_desc_match_mutual_f64.
//
// Arithmetic: fp64 with a fixed order and no contraction (__dadd_rn / __dmul_rn / __ddiv_rn / __dsqrt_rn), so that a
// float64 restatement on the host (tests/fgr_ref.py) follows every tuple, every sum and every solve.  The only steps
// that are not correctly rounded are the sin / cos of the pose update; see the header for the full rules.
#include "registration.cuh"

namespace usip {

constexpr int FGR_THREADS = 256;                 // also the tuple round: trials tested per round
constexpr int FGR_WARPS = FGR_THREADS / 32;
constexpr uint32_t FGR_PHILOX_TAG = 0x46475254u; // "FGRT"
constexpr int FGR_ITERATIONS = 640;
constexpr int FGR_TRIALS_PER_MATCH = 100;
constexpr int FGR_TUPLE_CAP = 10000;
constexpr int FGR_MIN_CORR = 10;
constexpr double FGR_DIV = 1.4, FGR_STOP = 0.05;
constexpr double FGR_SIM = (double)0.95f;        // the library's 0.95f, widened exactly
constexpr int FGR_NSUM = 27;                     // 21 of J^T J (upper triangle, row-major) and 6 of J^T r

struct FgrShared {
  double red[FGR_WARPS][FGR_NSUM];
  double T[12];                                  // the normalised-frame pose, row-major 3x4
  double delta[12];                              // this iteration's update [R_delta | t_delta]
  double mean[6];                                // fragment 1's mean, then fragment 2's
  unsigned long long scale_bits;                 // max centred norm (non-negative doubles order as their bits)
  double Rt[12];                                 // the de-normalised result
  int warp_tot[FGR_WARPS];
  int bad, nonfinite, stop, n_inl;
};

__device__ __forceinline__ double fgr_norm3(double x, double y, double z) {
  return __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(x, x), __dmul_rn(y, y)), __dmul_rn(z, z)));
}

// the 27 weighted terms of one correspondence (p, q) at scale par, weighted by its multiplicity w
__device__ __forceinline__ void fgr_terms(double px, double py, double pz, double qx, double qy, double qz, double par,
                                          double w, double out[FGR_NSUM]) {
  const double rx = dsub(px, qx), ry = dsub(py, qy), rz = dsub(pz, qz);
  const double rr = __dadd_rn(__dadd_rn(__dmul_rn(rx, rx), __dmul_rn(ry, ry)), __dmul_rn(rz, rz));
  const double t = __ddiv_rn(par, __dadd_rn(rr, par));
  const double ws = __dmul_rn(w, __dmul_rn(t, t));
  const double Jx[6] = {0.0, -qz, qy, -1.0, 0.0, 0.0};
  const double Jy[6] = {qz, 0.0, -qx, 0.0, -1.0, 0.0};
  const double Jz[6] = {-qy, qx, 0.0, 0.0, 0.0, -1.0};
  int e = 0;
#pragma unroll
  for (int a = 0; a < 6; ++a)
#pragma unroll
    for (int b = a; b < 6; ++b)
      out[e++] = __dmul_rn(__dadd_rn(__dadd_rn(__dmul_rn(Jx[a], Jx[b]), __dmul_rn(Jy[a], Jy[b])), __dmul_rn(Jz[a], Jz[b])),
                           ws);
#pragma unroll
  for (int a = 0; a < 6; ++a)
    out[21 + a] = __dmul_rn(__dadd_rn(__dadd_rn(__dmul_rn(Jx[a], rx), __dmul_rn(Jy[a], ry)), __dmul_rn(Jz[a], rz)), ws);
}

// Thread 0: Cholesky solve of J^T J xi = -J^T r and the update delta = [Rz(xi2) Ry(xi1) Rx(xi0) | xi3..5]; T = delta T.
// Returns false (T untouched) when a pivot is <= 0 or not finite.
__device__ bool fgr_solve_step(const double* S, double* T, double* delta) {
  double A[6][6], Lm[6][6], x[6];
  int e = 0;
#pragma unroll
  for (int a = 0; a < 6; ++a)
#pragma unroll
    for (int b = a; b < 6; ++b) { A[a][b] = S[e]; A[b][a] = S[e]; ++e; }
#pragma unroll
  for (int j = 0; j < 6; ++j) {
    double v = A[j][j];
#pragma unroll
    for (int k = 0; k < j; ++k) v = dsub(v, __dmul_rn(Lm[j][k], Lm[j][k]));
    if (!(v > 0.0 && v <= 1.7976931348623157e308)) return false;
    const double d = __dsqrt_rn(v);
    Lm[j][j] = d;
#pragma unroll
    for (int i = j + 1; i < 6; ++i) {
      double u = A[i][j];
#pragma unroll
      for (int k = 0; k < j; ++k) u = dsub(u, __dmul_rn(Lm[i][k], Lm[j][k]));
      Lm[i][j] = __ddiv_rn(u, d);
    }
  }
#pragma unroll
  for (int i = 0; i < 6; ++i) {                  // L y = -J^T r
    double v = -S[21 + i];
#pragma unroll
    for (int k = 0; k < i; ++k) v = dsub(v, __dmul_rn(Lm[i][k], x[k]));
    x[i] = __ddiv_rn(v, Lm[i][i]);
  }
#pragma unroll
  for (int i = 5; i >= 0; --i) {                 // L^T xi = y
    double v = x[i];
#pragma unroll
    for (int k = i + 1; k < 6; ++k) v = dsub(v, __dmul_rn(Lm[k][i], x[k]));
    x[i] = __ddiv_rn(v, Lm[i][i]);
  }
  const double sx = sin(x[0]), cx = cos(x[0]), sy = sin(x[1]), cy = cos(x[1]), sz = sin(x[2]), cz = cos(x[2]);
  const double czsy = __dmul_rn(cz, sy), szsy = __dmul_rn(sz, sy);
  double* D = delta;
  D[0] = __dmul_rn(cz, cy);
  D[1] = dsub(__dmul_rn(czsy, sx), __dmul_rn(sz, cx));
  D[2] = __dadd_rn(__dmul_rn(czsy, cx), __dmul_rn(sz, sx));
  D[3] = x[3];
  D[4] = __dmul_rn(sz, cy);
  D[5] = __dadd_rn(__dmul_rn(szsy, sx), __dmul_rn(cz, cx));
  D[6] = dsub(__dmul_rn(szsy, cx), __dmul_rn(cz, sx));
  D[7] = x[4];
  D[8] = -sy;
  D[9] = __dmul_rn(cy, sx);
  D[10] = __dmul_rn(cy, cx);
  D[11] = x[5];
  double N[12];
#pragma unroll
  for (int r = 0; r < 3; ++r) {
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const double v = __dadd_rn(__dadd_rn(__dmul_rn(D[4 * r], T[c]), __dmul_rn(D[4 * r + 1], T[4 + c])),
                                 __dmul_rn(D[4 * r + 2], T[8 + c]));
      N[4 * r + c] = c == 3 ? __dadd_rn(v, D[4 * r + 3]) : v;
    }
  }
  for (int i = 0; i < 12; ++i) T[i] = N[i];
  return true;
}

// One CTA per (pair, K).  Dynamic smem (cap entries each): the normalised points of the matches (p: fragment 1, q:
// fragment 2, SoA fp64; q is moved by every update; after the solve both hold the raw points), the multiplicities,
// the list of matches with a non-zero multiplicity, and the inlier flags.
__global__ void __launch_bounds__(FGR_THREADS)
fgr_kernel(const float* __restrict__ xyz, const int32_t* __restrict__ count, int L, const int32_t* __restrict__ pairs,
           RegKs ks, int nK, const int32_t* __restrict__ matches, const int32_t* __restrict__ n_matches, int cap,
           uint64_t seed, double thr, double* __restrict__ Rt_out, int32_t* __restrict__ n_tuples_out,
           int32_t* __restrict__ n_inl_out, double* __restrict__ info_out, int32_t* __restrict__ status_out) {
  extern __shared__ __align__(16) double fgr_smem[];
  __shared__ FgrShared sh;
  double* cpx = fgr_smem;
  double* cpy = cpx + cap;
  double* cpz = cpy + cap;
  double* cqx = cpz + cap;
  double* cqy = cqx + cap;
  double* cqz = cqy + cap;
  int32_t* mult = (int32_t*)(cqz + cap);
  int32_t* use = mult + cap;
  uint8_t* flag = (uint8_t*)(use + cap);
  const int pk = blockIdx.x, p = pk / nK, kk = pk % nK, tid = threadIdx.x;
  const int sa = pairs[2 * p], sp = pairs[2 * p + 1];
  const int K = ks.k[kk];
  const int n1 = min(min(count[sa], L), K), n2 = min(min(count[sp], L), K);
  const int npts = min(max(n_matches[pk], 0), cap);
  const int32_t* mt = matches + (int64_t)pk * cap * 2;
  const float* X1 = xyz + (int64_t)sa * L * 3;
  const float* X2 = xyz + (int64_t)sp * L * 3;

  if (tid == 0) { sh.bad = 0; sh.nonfinite = 0; sh.stop = 0; sh.n_inl = 0; sh.scale_bits = 0ull; }
  __syncthreads();
  for (int m = tid; m < npts; m += blockDim.x) {
    const int a = mt[2 * m], b = mt[2 * m + 1];
    if (a < 0 || a >= n1 || b < 0 || b >= n2) sh.bad = 1;
    mult[m] = 0;
  }
  // 1. NormalizePoints: each mean summed in row order, then / n; scale = max centred norm over both fragments
  if (tid < 6) {
    const float* X = tid < 3 ? X1 : X2;
    const int n = tid < 3 ? n1 : n2, c = tid % 3;
    double s = 0.0;
    for (int i = 0; i < n; ++i) s = __dadd_rn(s, (double)X[3 * i + c]);
    sh.mean[tid] = __ddiv_rn(s, (double)max(n, 1));
  }
  __syncthreads();
  if (sh.bad) {                                  // status 3: nothing computed
    if (tid < 36) info_out[(int64_t)pk * 36 + tid] = 0.0;
    if (tid < 12) Rt_out[(int64_t)pk * 12 + tid] = 0.0;
    if (tid == 0) { n_tuples_out[pk] = 0; n_inl_out[pk] = 0; status_out[pk] = 3; }
    return;
  }
  for (int i = tid; i < n1 + n2; i += blockDim.x) {
    const float* q = i < n1 ? X1 + 3 * i : X2 + 3 * (i - n1);
    const double* mu = i < n1 ? sh.mean : sh.mean + 3;
    const double r = fgr_norm3(dsub((double)q[0], mu[0]), dsub((double)q[1], mu[1]), dsub((double)q[2], mu[2]));
    if (!(r <= 1.7976931348623157e308)) sh.nonfinite = 1;
    else atomicMax(&sh.scale_bits, (unsigned long long)__double_as_longlong(r));
  }
  __syncthreads();
  const double scale = __longlong_as_double((long long)sh.scale_bits);
  const bool degenerate = sh.nonfinite || !(scale > 0.0);
  int status = degenerate ? 4 : 0, kept = 0;

  if (!degenerate) {
    for (int m = tid; m < npts; m += blockDim.x) {
      const int a = mt[2 * m], b = mt[2 * m + 1];
      cpx[m] = __ddiv_rn(dsub((double)X1[3 * a], sh.mean[0]), scale);
      cpy[m] = __ddiv_rn(dsub((double)X1[3 * a + 1], sh.mean[1]), scale);
      cpz[m] = __ddiv_rn(dsub((double)X1[3 * a + 2], sh.mean[2]), scale);
      cqx[m] = __ddiv_rn(dsub((double)X2[3 * b], sh.mean[3]), scale);
      cqy[m] = __ddiv_rn(dsub((double)X2[3 * b + 1], sh.mean[4]), scale);
      cqz[m] = __ddiv_rn(dsub((double)X2[3 * b + 2], sh.mean[5]), scale);
    }
    __syncthreads();
    // 3. the tuple test: trials in rounds of FGR_THREADS, the first FGR_TUPLE_CAP accepted in trial order are kept
    const int ntrial = npts >= 3 ? FGR_TRIALS_PER_MATCH * npts : 0;
    for (int base = 0; base < ntrial && kept < FGR_TUPLE_CAP; base += FGR_THREADS) {
      const int t = base + tid;
      bool acc = false;
      int idx[3] = {0, 0, 0};
      if (t < ntrial) {
        const uint4 r = philox4x32_10(make_uint4((uint32_t)t, 0u, FGR_PHILOX_TAG, 0u), (uint32_t)seed,
                                      (uint32_t)(seed >> 32));
        const double s32 = 2.3283064365386963e-10;                  // 2^-32
        const uint32_t w[3] = {r.x, r.y, r.z};
#pragma unroll
        for (int k = 0; k < 3; ++k)
          idx[k] = min((int)floor(__dmul_rn(__dmul_rn((double)w[k], s32), (double)npts)), npts - 1);
        acc = true;
#pragma unroll
        for (int k = 0; k < 3; ++k) {
          const int u = idx[k], v = idx[(k + 1) % 3];
          const double li = fgr_norm3(dsub(cpx[u], cpx[v]), dsub(cpy[u], cpy[v]), dsub(cpz[u], cpz[v]));
          const double lj = fgr_norm3(dsub(cqx[u], cqx[v]), dsub(cqy[u], cqy[v]), dsub(cqz[u], cqz[v]));
          acc = acc && __dmul_rn(li, FGR_SIM) < lj && lj < __ddiv_rn(li, FGR_SIM);
        }
      }
      int total;
      const int rank = reg_block_rank(acc, sh.warp_tot, &total);
      if (acc && kept + rank < FGR_TUPLE_CAP) {
        atomicAdd(&mult[idx[0]], 1); atomicAdd(&mult[idx[1]], 1); atomicAdd(&mult[idx[2]], 1);
      }
      kept = min(kept + total, FGR_TUPLE_CAP);
    }
    __syncthreads();
    if (3 * kept < FGR_MIN_CORR) status = 1;
  }

  if (status == 0) {
    // the matches in use: non-zero multiplicity, ascending
    int nuse = 0;
    for (int base = 0; base < npts; base += FGR_THREADS) {
      const int m = base + tid;
      const bool f = m < npts && mult[m] > 0;
      int total;
      const int at = nuse + reg_block_rank(f, sh.warp_tot, &total);
      if (f) use[at] = m;
      nuse += total;
    }
    if (tid < 12) sh.T[tid] = (tid % 5 == 0) ? 1.0 : 0.0;
    __syncthreads();
    // 4. graduated non-convexity
    double par = 1.0;
    const int lane = tid & 31, warp = tid >> 5;
    for (int itr = 0; itr < FGR_ITERATIONS; ++itr) {
      if (itr % 4 == 0 && par > FGR_STOP) par = __ddiv_rn(par, FGR_DIV);
      double acc[FGR_NSUM];
#pragma unroll
      for (int e = 0; e < FGR_NSUM; ++e) acc[e] = 0.0;
      for (int k = tid; k < nuse; k += FGR_THREADS) {
        const int m = use[k];
        double term[FGR_NSUM];
        fgr_terms(cpx[m], cpy[m], cpz[m], cqx[m], cqy[m], cqz[m], par, (double)mult[m], term);
#pragma unroll
        for (int e = 0; e < FGR_NSUM; ++e) acc[e] = __dadd_rn(acc[e], term[e]);
      }
#pragma unroll
      for (int e = 0; e < FGR_NSUM; ++e) {
        double v = acc[e];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v = __dadd_rn(v, __shfl_xor_sync(0xffffffffu, v, o));
        if (lane == 0) sh.red[warp][e] = v;
      }
      __syncthreads();
      if (tid == 0) {
        double S[FGR_NSUM];
#pragma unroll
        for (int e = 0; e < FGR_NSUM; ++e) {
          double v = sh.red[0][e];
          for (int w = 1; w < FGR_WARPS; ++w) v = __dadd_rn(v, sh.red[w][e]);
          S[e] = v;
        }
        if (!fgr_solve_step(S, sh.T, sh.delta)) sh.stop = 1;
      }
      __syncthreads();
      if (sh.stop) { status = 2; break; }
      for (int k = tid; k < nuse; k += FGR_THREADS) {
        const int m = use[k];
        double x = cqx[m], y = cqy[m], z = cqz[m];
        reg_map(sh.delta, x, y, z);
        cqx[m] = x; cqy[m] = y; cqz[m] = z;
      }
    }
  }

  __syncthreads();                               // the last update of q is done before the raw points replace it
  // 5. GetOutputTrans: R = T[:3, :3], t = ((-(R mean2)) + T[:3, 3] scale) + mean1
  if (tid == 0) {
    const bool moved = status == 0 || status == 2;
    const double sc = moved ? scale : 0.0;
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      double R[4];
#pragma unroll
      for (int c = 0; c < 4; ++c) R[c] = moved ? sh.T[4 * r + c] : (c == r ? 1.0 : 0.0);
      const double a = __dadd_rn(__dadd_rn(__dmul_rn(R[0], sh.mean[3]), __dmul_rn(R[1], sh.mean[4])),
                                 __dmul_rn(R[2], sh.mean[5]));
      sh.Rt[4 * r] = R[0]; sh.Rt[4 * r + 1] = R[1]; sh.Rt[4 * r + 2] = R[2];
      sh.Rt[4 * r + 3] = __dadd_rn(__dadd_rn(-a, __dmul_rn(R[3], sc)), sh.mean[r]);
    }
  }
  // the epilogue: inliers of every match under Rt, ascending, and the information matrix over them
  for (int m = tid; m < npts; m += blockDim.x) {
    const int a = mt[2 * m], b = mt[2 * m + 1];
    cpx[m] = (double)X1[3 * a]; cpy[m] = (double)X1[3 * a + 1]; cpz[m] = (double)X1[3 * a + 2];
    cqx[m] = (double)X2[3 * b]; cqy[m] = (double)X2[3 * b + 1]; cqz[m] = (double)X2[3 * b + 2];
  }
  __syncthreads();
  for (int m = tid; m < npts; m += blockDim.x) {
    const bool f = reg_inlier(sh.Rt, cpx[m], cpy[m], cpz[m], cqx[m], cqy[m], cqz[m], thr);
    flag[m] = f;
    if (f) atomicAdd(&sh.n_inl, 1);
  }
  __syncthreads();
  if (tid < 36) {
    const int r = tid / 6, c = tid % 6;
    double s = 0.0;
    for (int m = 0; m < npts; ++m)
      if (flag[m]) s = __dadd_rn(s, reg_info_entry(r, c, cpx[m], cpy[m], cpz[m]));
    info_out[(int64_t)pk * 36 + tid] = s;
  }
  if (tid < 12) Rt_out[(int64_t)pk * 12 + tid] = sh.Rt[tid];
  if (tid == 0) { n_tuples_out[pk] = kept; n_inl_out[pk] = sh.n_inl; status_out[pk] = status; }
}

}  // namespace usip

using namespace usip;

extern "C" int usip_fgr_f64(const float* xyz, const int32_t* count, int n_scans, int L, const int32_t* pairs, int P,
                            const int32_t* ks, int nK, const int32_t* matches, const int32_t* n_matches, int cap,
                            uint64_t seed, double threshold, double* Rt, int32_t* n_tuples, int32_t* n_inliers,
                            double* info, int32_t* status, void* stream) {
  USIP_REQUIRE(xyz && count && pairs && matches && n_matches && Rt && n_tuples && n_inliers && info && status,
               "fgr: null pointer");
  USIP_REQUIRE(n_scans > 0 && L > 0 && P > 0 && cap >= 1, "fgr: bad sizes");
  USIP_REQUIRE(L <= USIP_REG_MAX_KEYPOINTS, "fgr: more keypoints per scan than shared memory holds");
  USIP_REQUIRE(cap <= USIP_REG_MAX_KEYPOINTS, "fgr: match list longer than USIP_REG_MAX_KEYPOINTS");
  RegKs kk;
  if (int e = reg_check_ks(ks, nK, kk)) return e;
  USIP_REQUIRE(threshold > 0.0, "fgr: the inlier threshold must be > 0");
  const int smem = 6 * cap * (int)sizeof(double) + 2 * cap * (int)sizeof(int32_t) + ((cap + 15) / 16) * 16;
  cudaError_t e = cudaFuncSetAttribute(fgr_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  if (e != cudaSuccess) { set_last_error("fgr: smem attribute"); return (int)e; }
  fgr_kernel<<<P * nK, FGR_THREADS, smem, (cudaStream_t)stream>>>(xyz, count, L, pairs, kk, nK, matches, n_matches,
                                                                   cap, seed, threshold, Rt, n_tuples, n_inliers, info,
                                                                   status);
  return check_launch("fgr_kernel");
}
