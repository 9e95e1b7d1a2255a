/* ORACLE -- TEST INFRASTRUCTURE ONLY.  Never linked into libusip_b200.so and never on the product path.
 *
 * Plain-C CPU restatement of the integer/index parts of the USIP hot path.  Every function cites
 * the reference file:line it follows (paths relative to /root/reference).  Compile with
 *     gcc -O2 -fPIC -shared -ffp-contract=off -fno-fast-math
 * (-ffp-contract=off matters: the reference's distances are computed by separate ATen kernels
 * -- sub, mul, add, sqrt each rounded to fp32, no FMA -- verified by probing torch 2.11 CPU).
 *
 * Pinning: tests/test_oracle_vs_golden.py checks these functions against outputs of the real
 * reference (reference C++ forward_cpu compiled from its own sources + reference Python run on
 * CPU through oracle/ref_shim.py), frozen in tests/golden/.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

/* models/index_max_ext/index_max.cpp:73-112 (index_max_forward_cpu) -- identical semantics to the
 * CUDA kernels index_max_cuda.cu:9-25 and :29-61: max_val initialised to -1000, max_idx to 0,
 * strict '>' so the smallest n wins among equal maxima, values <= -1000 never win. */
void orc_index_max(const float* data, const int32_t* index, int32_t* max_idx,
                   int B, int C, int N, int K) {
  float* max_val = (float*)malloc(sizeof(float) * (size_t)K);
  for (int b = 0; b < B; ++b)
    for (int c = 0; c < C; ++c) {
      for (int k = 0; k < K; ++k) { max_val[k] = -1000.0f; max_idx[((size_t)b * C + c) * K + k] = 0; }
      const float* row = data + ((size_t)b * C + c) * N;
      for (int n = 0; n < N; ++n) {
        int k = index[(size_t)b * N + n];
        float v = row[n];
        if (v > max_val[k]) { max_val[k] = v; max_idx[((size_t)b * C + c) * K + k] = n; }
      }
    }
  free(max_val);
}

/* models/ball_query_ext/ball_query_cuda.cu:22-46: first K (ascending n) with dist <= radius;
 * 0 hits -> zeros; 0<u<K hits -> out[u+i] = out[i % u]. */
void orc_ball_query_dist(const float* dist, float radius, int32_t* out, int B, int M, int N, int K) {
  for (int b = 0; b < B; ++b)
    for (int m = 0; m < M; ++m) {
      const float* row = dist + ((size_t)b * M + m) * N;
      int32_t* o = out + ((size_t)b * M + m) * K;
      int u = 0;
      for (int n = 0; n < N && u < K; ++n)
        if (row[n] <= radius) o[u++] = n;
      if (u == 0) { for (int i = 0; i < K; ++i) o[i] = 0; }
      else if (u < K) { for (int i = 0; i < K - u; ++i) o[u + i] = o[i % u]; }
    }
}

/* fp32 distance exactly as the reference's ATen op sequence produces it:
 * diff = a - b; sq = diff*diff; s = (sq0 + sq1) + sq2   (util/som.py:35-36; probed) */
static inline float sqdist3(float ax, float ay, float az, float bx, float by, float bz) {
  float dx = ax - bx, dy = ay - by, dz = az - bz;
  float sx = dx * dx, sy = dy * dy, sz = dz * dz;
  float s = sx + sy;
  return s + sz;
}

/* models/networks.py:355-357 (torch.norm(node - pc, p=2, dim=1)) followed by
 * ball_query_cuda.cu:22-46.  xyz (B,3,N), centers (B,3,M). */
void orc_ball_query_xyz(const float* xyz, const float* centers, float radius, int32_t* out,
                        int B, int N, int M, int K) {
  for (int b = 0; b < B; ++b) {
    const float* px = xyz + (size_t)b * 3 * N; const float* py = px + N; const float* pz = py + N;
    const float* cx = centers + (size_t)b * 3 * M; const float* cy = cx + M; const float* cz = cy + M;
    for (int m = 0; m < M; ++m) {
      int32_t* o = out + ((size_t)b * M + m) * K;
      int u = 0;
      for (int n = 0; n < N && u < K; ++n) {
        float d = sqrtf(sqdist3(cx[m], cy[m], cz[m], px[n], py[n], pz[n]));
        if (d <= radius) o[u++] = n;
      }
      if (u == 0) { for (int i = 0; i < K; ++i) o[i] = 0; }
      else if (u < K) { for (int i = 0; i < K - u; ++i) o[u + i] = o[i % u]; }
    }
  }
}

/* util/som.py:35-39 with k=1: min_idx[b,n] = argmin_m sum_c (x - node)^2 (squared, no sqrt).
 * Ties resolve to the smallest m (what torch.topk(k=1,largest=False) returns on CPU; ties only
 * occur for duplicated nodes).  xyz (B,3,N), node (B,3,M) -> min_idx (B,N). */
void orc_som_assign(const float* xyz, const float* node, int32_t* min_idx, int B, int N, int M) {
  for (int b = 0; b < B; ++b) {
    const float* px = xyz + (size_t)b * 3 * N; const float* py = px + N; const float* pz = py + N;
    const float* nx = node + (size_t)b * 3 * M; const float* ny = nx + M; const float* nz = ny + M;
    for (int n = 0; n < N; ++n) {
      float best = INFINITY; int bi = 0;
      for (int m = 0; m < M; ++m) {
        float d = sqdist3(px[n], py[n], pz[n], nx[m], ny[m], nz[m]);
        if (d < best) { best = d; bi = m; }
      }
      min_idx[(size_t)b * N + n] = bi;
    }
  }
}

/* models/losses.py:62-66,134-141: d = torch.norm(a_i - b_j), min over j (first index on ties).
 * a (B,3,Ma), b (B,3,Nb) -> min_d (B,Ma), arg (B,Ma). */
void orc_pairwise_min(const float* a, const float* b, float* min_d, int32_t* arg, int B, int Ma, int Nb) {
  for (int bb = 0; bb < B; ++bb) {
    const float* ax = a + (size_t)bb * 3 * Ma; const float* ay = ax + Ma; const float* az = ay + Ma;
    const float* bx = b + (size_t)bb * 3 * Nb; const float* by = bx + Nb; const float* bz = by + Nb;
    for (int i = 0; i < Ma; ++i) {
      float best = INFINITY; int bi = 0;
      for (int j = 0; j < Nb; ++j) {
        float d = sqrtf(sqdist3(ax[i], ay[i], az[i], bx[j], by[j], bz[j]));
        if (d < best) { best = d; bi = j; }
      }
      min_d[(size_t)bb * Ma + i] = best; arg[(size_t)bb * Ma + i] = bi;
    }
  }
}

/* models/layers.py:417-421: norm = torch.norm(query - database, dim=1); topk(K, largest=False,
 * sorted=True).  Ascending distance, ties by ascending index.  query (B,3,M), db (B,3,N). */
void orc_knn(const float* query, const float* db, int32_t* knn_i, float* knn_d, int B, int M, int N, int K) {
  float* d = (float*)malloc(sizeof(float) * (size_t)N);
  uint8_t* used = (uint8_t*)malloc((size_t)N);
  for (int b = 0; b < B; ++b) {
    const float* qx = query + (size_t)b * 3 * M; const float* qy = qx + M; const float* qz = qy + M;
    const float* dx = db + (size_t)b * 3 * N; const float* dy = dx + N; const float* dz = dy + N;
    for (int m = 0; m < M; ++m) {
      for (int n = 0; n < N; ++n) { d[n] = sqrtf(sqdist3(qx[m], qy[m], qz[m], dx[n], dy[n], dz[n])); used[n] = 0; }
      for (int k = 0; k < K; ++k) {
        float best = INFINITY; int bi = -1;
        for (int n = 0; n < N; ++n) if (!used[n] && (bi < 0 || d[n] < best)) { best = d[n]; bi = n; }
        used[bi] = 1;
        knn_i[((size_t)b * M + m) * K + k] = bi;
        if (knn_d) knn_d[((size_t)b * M + m) * K + k] = best;
      }
    }
  }
  free(d); free(used);
}

/* data/kitti_detector_loader.py:68-83 (FarthestSampler.sample): the chosen set starts with pts[start]; the running
 * squared distance to the set is kept in float64 -- (p0 - pts)**2 summed over xyz left to right, p0 a float64 copy of a
 * float32 point -- and every further node is the FIRST arg-max of it (np.argmax).  pts (Ns,3) row-major. */
void orc_fps(const float* pts, int start, int32_t* out_idx, int Ns, int k) {
  double* dist = (double*)malloc(sizeof(double) * (size_t)Ns);
  int sel = start;
  for (int it = 0; it < k; ++it) {
    out_idx[it] = sel;
    if (it == k - 1) break;
    const double sx = pts[3 * sel], sy = pts[3 * sel + 1], sz = pts[3 * sel + 2];
    int best = 0;
    for (int n = 0; n < Ns; ++n) {
      const double dx = sx - (double)pts[3 * n], dy = sy - (double)pts[3 * n + 1], dz = sz - (double)pts[3 * n + 2];
      const double d = (dx * dx + dy * dy) + dz * dz;
      dist[n] = (it == 0 || d < dist[n]) ? d : dist[n];
      if (dist[n] > dist[best]) best = n;
    }
    sel = best;
  }
  free(dist);
}

/* evaluation/save_keypoints.py:180-216 nms(): kp (M,3) row-major, float32 np.linalg.norm distances, kept while
 * distance > radius; the next keypoint is always the FIRST arg-min of sigma among the remaining ones (np.argmin returns
 * the first NaN when there is one, so NaN sigmas go first, in index order).  Returns the number of kept keypoints, their
 * original indices in emission order in out_idx. */
int orc_nms(const float* kp, const float* sigma, float radius, int32_t* out_idx, int M) {
  if (radius < 0.01f) { for (int i = 0; i < M; ++i) out_idx[i] = i; return M; }
  uint8_t* gone = (uint8_t*)calloc((size_t)M, 1);
  int count = 0;
  for (;;) {
    int best = -1;
    for (int i = 0; i < M; ++i)
      if (!gone[i] && (best < 0 || (isnan(sigma[i]) && !isnan(sigma[best])) || sigma[i] < sigma[best])) best = i;
    if (best < 0) break;
    out_idx[count++] = best;
    for (int j = 0; j < M; ++j) {
      if (gone[j]) continue;
      const float d = sqrtf(sqdist3(kp[3 * best], kp[3 * best + 1], kp[3 * best + 2], kp[3 * j], kp[3 * j + 1], kp[3 * j + 2]));
      if (!(d > radius)) gone[j] = 1;
    }
  }
  free(gone);
  return count;
}
