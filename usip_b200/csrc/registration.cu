// registration.cu -- outdoor registration of evaluation/matlab/eval_outdoor (evaluate_kitti.m / evaluate_oxford.m):
// descriptor matching and RANSAC (external/ransacfitRt.m -> ransac.m, estimateRigidTransform.m) for every pair, every
// keypoint count K and every RANSAC trial budget of a sweep, two launches in all.
//
// Arithmetic: fp64 with a fixed order and no contraction (__dadd_rn / __dmul_rn / __ddiv_rn / __dsqrt_rn), so that a
// float64 restatement on the host (tests/reg_ref.py) reproduces every match, every hypothesis and every stop.  The
// only transcendental that decides anything is the log of ransac.m's trial estimate N; see the header.
#include "common.cuh"

namespace usip {

constexpr int REG_THREADS = 256;          // also the RANSAC chunk: hypotheses evaluated per round
constexpr int REG_JACOBI_SWEEPS = 8;
constexpr uint32_t REG_PHILOX_TAG = 0x52414e53u;

struct RegKs { int32_t k[USIP_REP_MAX_K]; };
struct RegTrials { int32_t t[USIP_REG_MAX_SWEEP]; };

__device__ __forceinline__ double dsub(double a, double b) { return __dadd_rn(a, -b); }

// ------------------------------------------------------------------------------------------------ matching
// Top-k of one query row against rows 0..n-1 of `set` (both (., D) f32), ordered by (d^2, index); d^2 is
// sum_c (q_c - s_c)^2 in fp64, c ascending, and a NaN d^2 (a non-finite descriptor value) counts as +inf.  The order is
// total and the slots start at (+inf, INT_MAX), so the first min(k, n) slots always hold real indices below n, whatever
// the values.  Rows are scanned in ascending index, so the lower index wins a tie.  Returns min(k, n).
template <int KMAX>
__device__ int reg_topk(const float* __restrict__ q, const float* __restrict__ set, int n, int D, int k, int* best) {
  const double inf = __longlong_as_double(0x7ff0000000000000ll);
  double bd[KMAX];
#pragma unroll
  for (int r = 0; r < KMAX; ++r) { bd[r] = inf; best[r] = 0x7fffffff; }
  for (int j = 0; j < n; ++j) {
    const float* s = set + (int64_t)j * D;
    double acc = 0.0;
    for (int c = 0; c < D; ++c) {
      const double d = dsub((double)__ldg(q + c), (double)__ldg(s + c));
      acc = __dadd_rn(acc, __dmul_rn(d, d));
    }
    // insertion: shift every entry that comes after (acc, j) one place down
    int bj = j;
    double bv = isnan(acc) ? inf : acc;
#pragma unroll
    for (int r = 0; r < KMAX; ++r) {
      if (r < k && (bv < bd[r] || (bv == bd[r] && bj < best[r]))) {
        const double tv = bd[r]; const int tj = best[r];
        bd[r] = bv; best[r] = bj; bv = tv; bj = tj;
      }
    }
  }
  return min(k, n);
}

// one CTA per (pair, K).  smem (k > 1): an na x np bitset of the union and the per-row counts.
__global__ void __launch_bounds__(REG_THREADS)
desc_match_kernel(const float* __restrict__ desc, const int32_t* __restrict__ count, int L, int D,
                  const int32_t* __restrict__ pairs, RegKs ks, int nK, int k, int cap, int32_t* __restrict__ matches,
                  int32_t* __restrict__ n_matches) {
  extern __shared__ __align__(16) uint32_t match_smem[];
  const int p = blockIdx.x / nK, kk = blockIdx.x % nK, tid = threadIdx.x;
  const int sa = pairs[2 * p], sp = pairs[2 * p + 1];
  const int K = ks.k[kk];
  const int na = min(min(count[sa], L), K), np = min(min(count[sp], L), K);
  const float* A = desc + (int64_t)sa * L * D;
  const float* Q = desc + (int64_t)sp * L * D;
  int32_t* out = matches + ((int64_t)p * nK + kk) * cap * 2;
  int best[8];

  if (k == 1) {
    for (int i = tid; i < na; i += blockDim.x) {
      reg_topk<1>(A + (int64_t)i * D, Q, np, D, 1, best);
      if (np > 0) { out[2 * i] = i; out[2 * i + 1] = best[0]; }
    }
    if (tid == 0) n_matches[(int64_t)p * nK + kk] = np > 0 ? na : 0;
    return;
  }

  const int W = (np + 31) >> 5;                                 // words per bitset row
  uint32_t* bits = match_smem;                                  // na * W
  int32_t* rowoff = (int32_t*)(bits + (size_t)L * ((L + 31) >> 5));   // na + 1
  for (int i = tid; i < na * W; i += blockDim.x) bits[i] = 0u;
  __syncthreads();
  for (int i = tid; i < na; i += blockDim.x) {                  // anchor i -> its k nearest positives
    const int n = reg_topk<8>(A + (int64_t)i * D, Q, np, D, k, best);
#pragma unroll
    for (int r = 0; r < 8; ++r)
      if (r < n && best[r] >= 0 && best[r] < np) atomicOr(&bits[i * W + (best[r] >> 5)], 1u << (best[r] & 31));
  }
  for (int j = tid; j < np; j += blockDim.x) {                  // positive j -> its k nearest anchors
    const int n = reg_topk<8>(Q + (int64_t)j * D, A, na, D, k, best);
#pragma unroll
    for (int r = 0; r < 8; ++r)
      if (r < n && best[r] >= 0 && best[r] < na) atomicOr(&bits[best[r] * W + (j >> 5)], 1u << (j & 31));
  }
  __syncthreads();
  for (int i = tid; i < na; i += blockDim.x) {
    int c = 0;
    for (int w = 0; w < W; ++w) c += __popc(bits[i * W + w]);
    rowoff[i + 1] = c;
  }
  __syncthreads();
  if (tid == 0) {
    rowoff[0] = 0;
    for (int i = 0; i < na; ++i) rowoff[i + 1] += rowoff[i];
    n_matches[(int64_t)p * nK + kk] = rowoff[na];
  }
  __syncthreads();
  for (int i = tid; i < na; i += blockDim.x) {                  // rows ascending by anchor, then positive: union(.., 'rows')
    int at = rowoff[i];
    for (int w = 0; w < W; ++w) {
      uint32_t b = bits[i * W + w];
      while (b) {
        const int j = (w << 5) + __ffs(b) - 1;
        b &= b - 1;
        out[2 * at] = i; out[2 * at + 1] = j;
        ++at;
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------ RANSAC
// Trial j's three uniforms: uploaded (row j of `uni`), or the first three words of Philox4x32-10 with counter
// (j, 0, tag, 0) and key (seed lo, seed hi), each times 2^-32.
__device__ __forceinline__ void reg_uniforms(const double* uni, int j, uint64_t seed, double u[3]) {
  if (uni) {
    u[0] = uni[3 * (int64_t)j]; u[1] = uni[3 * (int64_t)j + 1]; u[2] = uni[3 * (int64_t)j + 2];
    return;
  }
  const uint4 r = philox4x32_10(make_uint4((uint32_t)j, 0u, REG_PHILOX_TAG, 0u), (uint32_t)seed, (uint32_t)(seed >> 32));
  const double s = 2.3283064365386963e-10;                     // 2^-32
  u[0] = (double)r.x * s; u[1] = (double)r.y * s; u[2] = (double)r.z * s;
}

// three distinct indices below n (n >= 3), see the header
__device__ __forceinline__ void reg_pick3(const double u[3], int n, int idx[3]) {
  int i0 = min((int)floor(__dmul_rn(u[0], (double)n)), n - 1);
  int i1 = min((int)floor(__dmul_rn(u[1], (double)(n - 1))), n - 2);
  int i2 = min((int)floor(__dmul_rn(u[2], (double)(n - 2))), n - 3);
  i0 = max(i0, 0); i1 = max(i1, 0); i2 = max(i2, 0);
  if (i1 >= i0) ++i1;
  const int lo = min(i0, i1), hi = max(i0, i1);
  if (i2 >= lo) ++i2;
  if (i2 >= hi) ++i2;
  idx[0] = i0; idx[1] = i1; idx[2] = i2;
}

// A^T A for Horn's A of one centred correspondence (x: anchor, y: positive), estimateRigidTransform.m:
// A = [0, (y-x)^T; x-y, [y+x]_x]; entry (r, c) is ((A0r A0c + A1r A1c) + A2r A2c) + A3r A3c.
__device__ __forceinline__ void reg_ata(const double* x, const double* y, double M[4][4]) {
  const double u0 = dsub(y[0], x[0]), u1 = dsub(y[1], x[1]), u2 = dsub(y[2], x[2]);
  const double v0 = dsub(x[0], y[0]), v1 = dsub(x[1], y[1]), v2 = dsub(x[2], y[2]);
  const double w0 = __dadd_rn(y[0], x[0]), w1 = __dadd_rn(y[1], x[1]), w2 = __dadd_rn(y[2], x[2]);
  const double A[4][4] = {{0.0, u0, u1, u2}, {v0, 0.0, -w2, w1}, {v1, w2, 0.0, -w0}, {v2, -w1, w0, 0.0}};
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int c = 0; c < 4; ++c)
      M[r][c] = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(A[0][r], A[0][c]), __dmul_rn(A[1][r], A[1][c])),
                                    __dmul_rn(A[2][r], A[2][c])), __dmul_rn(A[3][r], A[3][c]));
}

// entry (r, c) of the same product, for a runtime (r, c): column r of A is selected, not indexed
__device__ __forceinline__ double reg_ata_entry(const double* x, const double* y, int r, int c) {
  const double u0 = dsub(y[0], x[0]), u1 = dsub(y[1], x[1]), u2 = dsub(y[2], x[2]);
  const double v0 = dsub(x[0], y[0]), v1 = dsub(x[1], y[1]), v2 = dsub(x[2], y[2]);
  const double w0 = __dadd_rn(y[0], x[0]), w1 = __dadd_rn(y[1], x[1]), w2 = __dadd_rn(y[2], x[2]);
  double col[2][4];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int k = h ? c : r;
    col[h][0] = k == 0 ? 0.0 : k == 1 ? u0 : k == 2 ? u1 : u2;
    col[h][1] = k == 0 ? v0 : k == 1 ? 0.0 : k == 2 ? -w2 : w1;
    col[h][2] = k == 0 ? v1 : k == 1 ? w2 : k == 2 ? 0.0 : -w0;
    col[h][3] = k == 0 ? v2 : k == 1 ? -w1 : k == 2 ? w0 : 0.0;
  }
  return __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(col[0][0], col[1][0]), __dmul_rn(col[0][1], col[1][1])),
                             __dmul_rn(col[0][2], col[1][2])), __dmul_rn(col[0][3], col[1][3]));
}

// Smallest eigenvector of the symmetric B (cyclic Jacobi, pairs (0,1) (0,2) (0,3) (1,2) (1,3) (2,3), a fixed number
// of sweeps, a rotation skipped when its off-diagonal entry is exactly 0) -> quat2rot.m without normalisation ->
// R; t = xbar - R ybar.  Rt row-major (3, 4).
__device__ __forceinline__ void reg_horn_finish(double a[4][4], const double* xbar, const double* ybar, double* Rt) {
  double V[4][4];
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int c = 0; c < 4; ++c) V[r][c] = r == c ? 1.0 : 0.0;
  constexpr int PP[6] = {0, 0, 0, 1, 1, 2}, QQ[6] = {1, 2, 3, 2, 3, 3};
  for (int sw = 0; sw < REG_JACOBI_SWEEPS; ++sw) {
#pragma unroll
    for (int e = 0; e < 6; ++e) {
      const int p = PP[e], q = QQ[e];
      const double apq = a[p][q];
      if (apq == 0.0) continue;
      const double theta = __ddiv_rn(dsub(a[q][q], a[p][p]), __dmul_rn(2.0, apq));
      const double at = fabs(theta);
      const double den = __dadd_rn(at, __dsqrt_rn(__dadd_rn(__dmul_rn(theta, theta), 1.0)));
      const double t = __ddiv_rn(theta >= 0.0 ? 1.0 : -1.0, den);
      const double c = __ddiv_rn(1.0, __dsqrt_rn(__dadd_rn(__dmul_rn(t, t), 1.0)));
      const double s = __dmul_rn(t, c);
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        if (r == p || r == q) continue;
        const double arp = a[r][p], arq = a[r][q];
        const double np_ = dsub(__dmul_rn(c, arp), __dmul_rn(s, arq));
        const double nq_ = __dadd_rn(__dmul_rn(s, arp), __dmul_rn(c, arq));
        a[r][p] = np_; a[p][r] = np_; a[r][q] = nq_; a[q][r] = nq_;
      }
      a[p][p] = dsub(a[p][p], __dmul_rn(t, apq));
      a[q][q] = __dadd_rn(a[q][q], __dmul_rn(t, apq));
      a[p][q] = 0.0; a[q][p] = 0.0;
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        const double vp = V[r][p], vq = V[r][q];
        V[r][p] = dsub(__dmul_rn(c, vp), __dmul_rn(s, vq));
        V[r][q] = __dadd_rn(__dmul_rn(s, vp), __dmul_rn(c, vq));
      }
    }
  }
  int m = 0;
  double amin = a[0][0];
#pragma unroll
  for (int r = 1; r < 4; ++r)
    if (a[r][r] < amin) { amin = a[r][r]; m = r; }
  double q0 = V[0][0], q1 = V[1][0], q2 = V[2][0], q3 = V[3][0];
#pragma unroll
  for (int r = 1; r < 4; ++r)
    if (m == r) { q0 = V[0][r]; q1 = V[1][r]; q2 = V[2][r]; q3 = V[3][r]; }
  const double s00 = __dmul_rn(q0, q0), s11 = __dmul_rn(q1, q1), s22 = __dmul_rn(q2, q2), s33 = __dmul_rn(q3, q3);
  double R[9];
  R[0] = dsub(dsub(__dadd_rn(s00, s11), s22), s33);
  R[1] = __dmul_rn(2.0, dsub(__dmul_rn(q1, q2), __dmul_rn(q0, q3)));
  R[2] = __dmul_rn(2.0, __dadd_rn(__dmul_rn(q1, q3), __dmul_rn(q0, q2)));
  R[3] = __dmul_rn(2.0, __dadd_rn(__dmul_rn(q1, q2), __dmul_rn(q0, q3)));
  R[4] = dsub(__dadd_rn(dsub(s00, s11), s22), s33);
  R[5] = __dmul_rn(2.0, dsub(__dmul_rn(q2, q3), __dmul_rn(q0, q1)));
  R[6] = __dmul_rn(2.0, dsub(__dmul_rn(q1, q3), __dmul_rn(q0, q2)));
  R[7] = __dmul_rn(2.0, __dadd_rn(__dmul_rn(q2, q3), __dmul_rn(q0, q1)));
  R[8] = __dadd_rn(dsub(dsub(s00, s11), s22), s33);
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    Rt[4 * r] = R[3 * r]; Rt[4 * r + 1] = R[3 * r + 1]; Rt[4 * r + 2] = R[3 * r + 2];
    const double ry = __dadd_rn(__dadd_rn(__dmul_rn(R[3 * r], ybar[0]), __dmul_rn(R[3 * r + 1], ybar[1])),
                                __dmul_rn(R[3 * r + 2], ybar[2]));
    Rt[4 * r + 3] = dsub(xbar[r], ry);
  }
}

// Horn's fit of three correspondences in sample order (the hypothesis of one trial)
__device__ __forceinline__ void reg_fit3(const double (*x)[3], const double (*y)[3], double* Rt) {
  double xb[3], yb[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    xb[c] = __ddiv_rn(__dadd_rn(__dadd_rn(__dadd_rn(0.0, x[0][c]), x[1][c]), x[2][c]), 3.0);
    yb[c] = __ddiv_rn(__dadd_rn(__dadd_rn(__dadd_rn(0.0, y[0][c]), y[1][c]), y[2][c]), 3.0);
  }
  double xc[3][3], yc[3][3];
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int c = 0; c < 3; ++c) { xc[i][c] = dsub(x[i][c], xb[c]); yc[i][c] = dsub(y[i][c], yb[c]); }
  double B[4][4], M[4][4];
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int c = 0; c < 4; ++c) B[r][c] = 0.0;
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    reg_ata(xc[i], yc[i], M);
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int c = 0; c < 4; ++c) B[r][c] = __dadd_rn(B[r][c], M[r][c]);
  }
  reg_horn_finish(B, xb, yb, Rt);
}

// ||x1 - (R x2 + t)|| < thr, each row ((R0 x + R1 y) + R2 z) + t, then ((dx^2 + dy^2) + dz^2), sqrt
__device__ __forceinline__ bool reg_inlier(const double* Rt, double ax, double ay, double az, double px, double py,
                                           double pz, double thr) {
  const double ex = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(Rt[0], px), __dmul_rn(Rt[1], py)), __dmul_rn(Rt[2], pz)), Rt[3]);
  const double ey = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(Rt[4], px), __dmul_rn(Rt[5], py)), __dmul_rn(Rt[6], pz)), Rt[7]);
  const double ez = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(Rt[8], px), __dmul_rn(Rt[9], py)), __dmul_rn(Rt[10], pz)), Rt[11]);
  const double dx = dsub(ax, ex), dy = dsub(ay, ey), dz = dsub(az, ez);
  return __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz))) < thr;
}

// ((m0*x + m1*y) + m2*z) + m3 for the three rows of a row-major 3x4 map (repeatability.cu's order)
__device__ __forceinline__ void reg_map(const double* T, double& x, double& y, double& z) {
  const double a = x, b = y, c = z;
  x = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(T[0], a), __dmul_rn(T[1], b)), __dmul_rn(T[2], c)), T[3]);
  y = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(T[4], a), __dmul_rn(T[5], b)), __dmul_rn(T[6], c)), T[7]);
  z = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(T[8], a), __dmul_rn(T[9], b)), __dmul_rn(T[10], c)), T[11]);
}

struct RegShared {                          // the static part of the RANSAC kernel's shared memory
  int32_t cnt[REG_THREADS];
  double Rt[12];
  double cen[6];
  double B[16];
  int32_t snap_tc[USIP_REG_MAX_SWEEP], snap_best[USIP_REG_MAX_SWEEP], snap_n[USIP_REG_MAX_SWEEP];
  int32_t trials[USIP_REG_MAX_SWEEP];
  int32_t done, bad;
};

// one CTA per (pair, K); dynamic smem: anchor and positive points (SoA fp64, L each), the match list (anchor | pos
// << 16) and the inlier flags of the refit
__global__ void __launch_bounds__(REG_THREADS)
ransac_kernel(const float* __restrict__ xyz, const int32_t* __restrict__ count, int L,
              const int32_t* __restrict__ pairs, const double* __restrict__ frames, int nK,
              const int32_t* __restrict__ matches, const int32_t* __restrict__ n_matches, int cap, RegTrials trials,
              int nT, double thr, uint64_t seed, const double* __restrict__ uni, double* __restrict__ Rt_out,
              int32_t* __restrict__ n_inl_out, int32_t* __restrict__ tc_out, int32_t* __restrict__ best_out,
              int32_t* __restrict__ status_out) {
  extern __shared__ __align__(16) double reg_smem[];
  __shared__ RegShared sh;
  double* ax = reg_smem;
  double* ay = ax + L;
  double* az = ay + L;
  double* px = az + L;
  double* py = px + L;
  double* pz = py + L;
  uint32_t* mi = (uint32_t*)(pz + L);
  uint8_t* flag = (uint8_t*)(mi + cap);
  const int pk = blockIdx.x, p = pk / nK, tid = threadIdx.x;
  const int sa = pairs[2 * p], sp = pairs[2 * p + 1];
  const int na = min(count[sa], L), np = min(count[sp], L);
  const int npts = min(max(n_matches[pk], 0), cap);
  const double* F = frames + (int64_t)p * 36;
  const int64_t ob = (int64_t)pk * nT;

  if (tid == 0) { sh.done = 0; sh.bad = 0; }
  if (tid < nT) sh.trials[tid] = trials.t[tid];
  for (int i = tid; i < na; i += blockDim.x) {
    const float* q = xyz + ((int64_t)sa * L + i) * 3;
    double x = q[0], y = q[1], z = q[2];
    reg_map(F, x, y, z);
    ax[i] = x; ay[i] = y; az[i] = z;
  }
  for (int i = tid; i < np; i += blockDim.x) {
    const float* q = xyz + ((int64_t)sp * L + i) * 3;
    double x = q[0], y = q[1], z = q[2];
    reg_map(F + 12, x, y, z);
    px[i] = x; py[i] = y; pz[i] = z;
  }
  __syncthreads();
  for (int m = tid; m < npts; m += blockDim.x) {
    const int a = matches[((int64_t)pk * cap + m) * 2], b = matches[((int64_t)pk * cap + m) * 2 + 1];
    if (a < 0 || a >= na || b < 0 || b >= np) { sh.bad = 1; mi[m] = 0; }
    else mi[m] = (uint32_t)a | ((uint32_t)b << 16);
  }
  __syncthreads();
  if (sh.bad || npts < 3) {
    if (tid < nT) {
      for (int e = 0; e < 12; ++e) Rt_out[(ob + tid) * 12 + e] = 0.0;
      n_inl_out[ob + tid] = 0; tc_out[ob + tid] = 0; best_out[ob + tid] = -1;
      status_out[ob + tid] = sh.bad ? 3 : 1;
    }
    return;
  }

  if (npts > 3) {
    // ransac.m's loop, one chunk of REG_THREADS trials per round; thread 0 replays the sequential update in trial order
    const int tmax = sh.trials[nT - 1];
    const double log_1mp = log(dsub(1.0, 0.99));
    const double eps = 2.220446049250313e-16;
    int trialcount = 0, best = -1, bestscore = 0, settled = 0;
    double N = 1.0;
    for (int base = 0; !sh.done; base += REG_THREADS) {
      const int j = base + tid;
      int c = -1;
      if (j <= tmax) {
        double u[3]; int idx[3]; double x[3][3], y[3][3], Rt[12];
        reg_uniforms(uni, j, seed, u);
        reg_pick3(u, npts, idx);
#pragma unroll
        for (int s = 0; s < 3; ++s) {
          const uint32_t w = mi[idx[s]];
          const int a = w & 0xffff, b = w >> 16;
          x[s][0] = ax[a]; x[s][1] = ay[a]; x[s][2] = az[a];
          y[s][0] = px[b]; y[s][1] = py[b]; y[s][2] = pz[b];
        }
        reg_fit3(x, y, Rt);
        c = 0;
        for (int m = 0; m < npts; ++m) {
          const uint32_t w = mi[m];
          const int a = w & 0xffff, b = w >> 16;
          c += reg_inlier(Rt, ax[a], ay[a], az[a], px[b], py[b], pz[b], thr);
        }
      }
      sh.cnt[tid] = c;
      __syncthreads();
      if (tid == 0) {
        for (int r = 0; r < REG_THREADS && settled < nT; ++r) {
          const int n = sh.cnt[r];
          if (n >= bestscore) {
            bestscore = n; best = base + r;
            const double frac = __ddiv_rn((double)n, (double)npts);
            double pno = dsub(1.0, __dmul_rn(__dmul_rn(frac, frac), frac));
            pno = fmin(fmax(eps, pno), dsub(1.0, eps));
            N = fmax(__ddiv_rn(log_1mp, log(pno)), 10.0);
          }
          ++trialcount;
          const bool stop = !(N > (double)trialcount);
          while (settled < nT && (stop || trialcount > sh.trials[settled])) {
            sh.snap_tc[settled] = trialcount; sh.snap_best[settled] = best; sh.snap_n[settled] = bestscore;
            ++settled;
          }
        }
        if (settled == nT) sh.done = 1;
      }
      __syncthreads();
    }
  }

  // finish: refit each sweep value's best inlier set (ransacfitRt.m); consecutive values that share a best trial share
  // the result
  for (int T = 0; T < nT; ++T) {
    const int b = npts == 3 ? -1 : sh.snap_best[T];
    const int64_t o = ob + T;
    if (T > 0 && (npts == 3 || b == sh.snap_best[T - 1])) {
      if (tid < 12) Rt_out[o * 12 + tid] = Rt_out[(o - 1) * 12 + tid];
      if (tid == 0) {
        n_inl_out[o] = n_inl_out[o - 1]; best_out[o] = b; status_out[o] = status_out[o - 1];
        tc_out[o] = npts == 3 ? 0 : sh.snap_tc[T];
      }
      continue;
    }
    if (npts == 3) {
      for (int m = tid; m < 3; m += blockDim.x) flag[m] = 1;
    } else {
      if (tid == 0) {
        double u[3]; int idx[3]; double x[3][3], y[3][3];
        reg_uniforms(uni, b, seed, u);
        reg_pick3(u, npts, idx);
#pragma unroll
        for (int s = 0; s < 3; ++s) {
          const uint32_t w = mi[idx[s]];
          const int a = w & 0xffff, c = w >> 16;
          x[s][0] = ax[a]; x[s][1] = ay[a]; x[s][2] = az[a];
          y[s][0] = px[c]; y[s][1] = py[c]; y[s][2] = pz[c];
        }
        reg_fit3(x, y, sh.Rt);
      }
      __syncthreads();
      for (int m = tid; m < npts; m += blockDim.x) {
        const uint32_t w = mi[m];
        const int a = w & 0xffff, c = w >> 16;
        flag[m] = reg_inlier(sh.Rt, ax[a], ay[a], az[a], px[c], py[c], pz[c], thr);
      }
    }
    __syncthreads();
    const int ninl = npts == 3 ? 3 : sh.snap_n[T];
    if (ninl >= 3) {
      if (tid < 6) {                                    // centroids, sum over the inliers in list order, then / n
        double s = 0.0;
        for (int m = 0; m < npts; ++m) {
          if (!flag[m]) continue;
          const uint32_t w = mi[m];
          const int i = tid < 3 ? (int)(w & 0xffff) : (int)(w >> 16);
          const double* col = tid < 3 ? (tid == 0 ? ax : tid == 1 ? ay : az) : (tid == 3 ? px : tid == 4 ? py : pz);
          s = __dadd_rn(s, col[i]);
        }
        sh.cen[tid] = __ddiv_rn(s, (double)ninl);
      }
      __syncthreads();
      if (tid < 16) {                                   // B entry tid, summed over the inliers in list order
        double s = 0.0;
        for (int m = 0; m < npts; ++m) {
          if (!flag[m]) continue;
          const uint32_t w = mi[m];
          const int a = w & 0xffff, q = w >> 16;
          const double x[3] = {dsub(ax[a], sh.cen[0]), dsub(ay[a], sh.cen[1]), dsub(az[a], sh.cen[2])};
          const double y[3] = {dsub(px[q], sh.cen[3]), dsub(py[q], sh.cen[4]), dsub(pz[q], sh.cen[5])};
          s = __dadd_rn(s, reg_ata_entry(x, y, tid >> 2, tid & 3));
        }
        sh.B[tid] = s;
      }
      __syncthreads();
    }
    if (tid == 0) {
      double* R = Rt_out + o * 12;
      if (ninl >= 3) {
        double Bm[4][4], Rt[12];
#pragma unroll
        for (int e = 0; e < 16; ++e) Bm[e >> 2][e & 3] = sh.B[e];
        reg_horn_finish(Bm, sh.cen, sh.cen + 3, Rt);
#pragma unroll
        for (int e = 0; e < 12; ++e) R[e] = Rt[e];
      } else {
        for (int e = 0; e < 12; ++e) R[e] = 0.0;
      }
      n_inl_out[o] = ninl; best_out[o] = b; status_out[o] = ninl >= 3 ? 0 : 2;
      tc_out[o] = npts == 3 ? 0 : sh.snap_tc[T];
    }
    __syncthreads();
  }
}

__global__ void ransac_uniforms_kernel(uint64_t seed, int T, double* __restrict__ out) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= T) return;
  double u[3];
  reg_uniforms(nullptr, j, seed, u);
  out[3 * (int64_t)j] = u[0]; out[3 * (int64_t)j + 1] = u[1]; out[3 * (int64_t)j + 2] = u[2];
}

int reg_check_ks(const int32_t* ks, int nK, RegKs& k) {
  USIP_REQUIRE(ks && nK >= 1 && nK <= USIP_REP_MAX_K, "registration: 1 to USIP_REP_MAX_K keypoint counts");
  for (int i = 0; i < nK; ++i) {
    USIP_REQUIRE(ks[i] > 0 && (i == 0 || ks[i] > ks[i - 1]), "registration: keypoint counts must ascend and be > 0");
    k.k[i] = ks[i];
  }
  return 0;
}

}  // namespace usip

using namespace usip;

extern "C" int usip_desc_match_f64(const float* desc, const int32_t* count, int n_scans, int L, int D,
                                   const int32_t* pairs, int P, const int32_t* ks, int nK, int k, int32_t* matches,
                                   int32_t* n_matches, void* stream) {
  USIP_REQUIRE(desc && count && pairs && matches && n_matches, "desc_match: null pointer");
  USIP_REQUIRE(n_scans > 0 && L > 0 && D > 0 && P > 0, "desc_match: bad sizes");
  USIP_REQUIRE(D <= USIP_REG_MAX_DIM, "desc_match: descriptor length over USIP_REG_MAX_DIM");
  USIP_REQUIRE(L <= USIP_REG_MAX_KEYPOINTS, "desc_match: more keypoints per scan than shared memory holds");
  USIP_REQUIRE(k >= 1 && k <= USIP_REG_MAX_MATCH_K, "desc_match: k must be 1 (one-way 1-NN) or 2..8 (k-NN union)");
  RegKs kk;
  if (int e = reg_check_ks(ks, nK, kk)) return e;
  const int cap = k == 1 ? L : 2 * k * L;
  const int smem = k == 1 ? 0 : (L * ((L + 31) / 32) + L + 1) * (int)sizeof(uint32_t);
  cudaError_t e = cudaFuncSetAttribute(desc_match_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  if (e != cudaSuccess) { set_last_error("desc_match: smem attribute"); return (int)e; }
  desc_match_kernel<<<P * nK, REG_THREADS, smem, (cudaStream_t)stream>>>(desc, count, L, D, pairs, kk, nK, k, cap,
                                                                         matches, n_matches);
  return check_launch("desc_match_kernel");
}

extern "C" int usip_ransac_rt_f64(const float* xyz, const int32_t* count, int n_scans, int L, const int32_t* pairs,
                                  const double* frames, int P, int nK, const int32_t* matches,
                                  const int32_t* n_matches, int cap, const int32_t* trials, int nT, double threshold,
                                  uint64_t seed, const double* uniforms, double* Rt, int32_t* n_inliers,
                                  int32_t* trialcount, int32_t* best_trial, int32_t* status, void* stream) {
  USIP_REQUIRE(xyz && count && pairs && frames && matches && n_matches && trials && Rt && n_inliers && trialcount &&
               best_trial && status, "ransac: null pointer");
  USIP_REQUIRE(n_scans > 0 && L > 0 && P > 0 && nK >= 1 && nK <= USIP_REP_MAX_K && cap >= 1, "ransac: bad sizes");
  USIP_REQUIRE(L <= USIP_REG_MAX_KEYPOINTS, "ransac: more keypoints per scan than shared memory holds");
  USIP_REQUIRE(cap <= 2 * USIP_REG_MAX_MATCH_K * L, "ransac: match list longer than 2 * 8 * L");
  USIP_REQUIRE(nT >= 1 && nT <= USIP_REG_MAX_SWEEP, "ransac: 1 to USIP_REG_MAX_SWEEP trial budgets");
  RegTrials t;
  for (int i = 0; i < nT; ++i) {
    USIP_REQUIRE(trials[i] >= 1 && trials[i] <= USIP_REG_MAX_TRIALS && (i == 0 || trials[i] > trials[i - 1]),
                 "ransac: trial budgets must ascend, be >= 1 and <= USIP_REG_MAX_TRIALS");
    t.t[i] = trials[i];
  }
  USIP_REQUIRE(threshold > 0.0, "ransac: the inlier threshold must be > 0");
  const int smem = 6 * L * (int)sizeof(double) + cap * (int)sizeof(uint32_t) + ((cap + 15) / 16) * 16;
  cudaError_t e = cudaFuncSetAttribute(ransac_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  if (e != cudaSuccess) { set_last_error("ransac: smem attribute"); return (int)e; }
  ransac_kernel<<<P * nK, REG_THREADS, smem, (cudaStream_t)stream>>>(xyz, count, L, pairs, frames, nK, matches,
                                                                     n_matches, cap, t, nT, threshold, seed, uniforms,
                                                                     Rt, n_inliers, trialcount, best_trial, status);
  return check_launch("ransac_kernel");
}

extern "C" int usip_ransac_uniforms(uint64_t seed, int T, double* out, void* stream) {
  USIP_REQUIRE(out && T > 0, "ransac_uniforms: bad arguments");
  ransac_uniforms_kernel<<<cdiv(T, 256), 256, 0, (cudaStream_t)stream>>>(seed, T, out);
  return check_launch("ransac_uniforms_kernel");
}
