/*
 * oracle_ransac.c -- CPU restatement of [O3D] v0.15.1 RegistrationRANSACBasedOnFeatureMatching as PlaceRecognition::
 * buildLoopClosureConstraints calls it (core/src/PlaceRecognition.cpp:81-86), rules 1-7 of DESIGN.md row K-ransac, one hypothesis
 * after the other.  TEST INFRASTRUCTURE ONLY: the ground truth of the device path in ransac.cu.  The 1-NN of the validation is the
 * oracle's KD-tree (orc_kdtree_search_hybrid), the SVD the oracle's orc_svd3.  Restated from the published algorithm (Open3D's
 * source is not available here).  Compiled with -ffp-contract=off: every expression is evaluated as written.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

void* orc_kdtree_build(const double* pts, int n);
void orc_kdtree_free(void* t);
int orc_kdtree_search_hybrid(void* t, const double* q, double radius, int max_nn, double* d2, int* idx);
void orc_svd3(const double* A, double* U, double* S, double* V);

#define MAX_N 8

/* rule 1: exact argmin both ways, d2 summed over k ascending, ties to the lower index; -1 when the other side is empty */
void or_feature_corr(const double* fs, int ns, const double* ft, int nt, int* s2t, int* t2s) {
  double* bt = (double*)malloc(sizeof(double) * (size_t)(nt > 0 ? nt : 1));
  for (int j = 0; j < nt; j++) { bt[j] = INFINITY; t2s[j] = -1; }
  for (int i = 0; i < ns; i++) {
    double bd = INFINITY; int bj = -1;
    for (int j = 0; j < nt; j++) {
      double d = 0.0;
      for (int k = 0; k < 33; k++) { const double e = fs[33 * (size_t)i + k] - ft[33 * (size_t)j + k]; d = d + e * e; }
      if (d < bd) { bd = d; bj = j; }
      if (d < bt[j]) { bt[j] = d; t2s[j] = i; }
    }
    s2t[i] = bj;
  }
  free(bt);
}

static uint64_t splitmix64(uint64_t z) {
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

/* rule 3: idx(h, j) = mulhi64(splitmix64(seed + (h n + j + 1) 0x9E3779B97F4A7C15), size) */
uint64_t or_stream(uint64_t seed, int64_t h, int n, int j, uint64_t size) {
  const uint64_t u = splitmix64(seed + (uint64_t)(h * n + j + 1) * 0x9E3779B97F4A7C15ull);
  return (uint64_t)(((unsigned __int128)u * size) >> 64);
}

static double norm3(double x, double y, double z) { return sqrt(x * x + y * y + z * z); }
static double det3(const double* M) {
  return M[0] * (M[4] * M[8] - M[5] * M[7]) - M[1] * (M[3] * M[8] - M[5] * M[6]) + M[2] * (M[3] * M[7] - M[4] * M[6]);
}
static void xform(const double* T, const double* p, double* o) {
  o[0] = ((T[0] * p[0] + T[1] * p[1]) + T[2] * p[2]) + T[3];
  o[1] = ((T[4] * p[0] + T[5] * p[1]) + T[6] * p[2]) + T[7];
  o[2] = ((T[8] * p[0] + T[9] * p[1]) + T[10] * p[2]) + T[11];
}

/* rule 4: Eigen::umeyama without scaling, two passes (means, then the demeaned covariance times 1/n) */
static void umeyama(const double S[][3], const double Q[][3], int n, double* T) {
  const double one_over_n = 1.0 / (double)n;
  double ms[3] = {0, 0, 0}, mt[3] = {0, 0, 0}, sigma[9] = {0};
  for (int j = 0; j < n; j++) for (int a = 0; a < 3; a++) { ms[a] += S[j][a]; mt[a] += Q[j][a]; }
  for (int a = 0; a < 3; a++) { ms[a] *= one_over_n; mt[a] *= one_over_n; }
  for (int j = 0; j < n; j++) for (int a = 0; a < 3; a++) for (int b = 0; b < 3; b++) sigma[3 * a + b] += (Q[j][a] - mt[a]) * (S[j][b] - ms[b]);
  for (int a = 0; a < 9; a++) sigma[a] *= one_over_n;
  double U[9], Sv[3], V[9], R[9];
  orc_svd3(sigma, U, Sv, V);
  const double sgn = det3(U) * det3(V) < 0 ? -1.0 : 1.0;
  for (int a = 0; a < 3; a++) for (int b = 0; b < 3; b++) R[3 * a + b] = U[3 * a] * V[3 * b] + U[3 * a + 1] * V[3 * b + 1] + sgn * U[3 * a + 2] * V[3 * b + 2];
  for (int i = 0; i < 16; i++) T[i] = (i % 5 == 0) ? 1.0 : 0.0;
  for (int a = 0; a < 3; a++) {
    for (int b = 0; b < 3; b++) T[4 * a + b] = R[3 * a + b];
    T[4 * a + 3] = mt[a] - (R[3 * a] * ms[0] + R[3 * a + 1] * ms[1] + R[3 * a + 2] * ms[2]);
  }
}

/* stats: [0] hypotheses (the h the loop stopped at), [1] validations, [2] |set|, [3] used_mutual, [4] best h (-1 = empty),
 *        [5] inliers.  sums: [0] sum d2 of best, [1] fitness, [2] rmse, [3] k_d of the last update.  T: 16 doubles. */
void or_ransac(const double* sx, const double* sf, int ns, const double* tx, const double* tf, int nt, int mutual_filter, int n,
               double max_corr, double checker_dist, double checker_edge, int64_t max_iteration, double confidence, uint64_t seed,
               double* T_out, int64_t* stats, double* sums) {
  for (int i = 0; i < 16; i++) T_out[i] = (i % 5 == 0) ? 1.0 : 0.0;
  memset(stats, 0, 6 * sizeof(int64_t)); stats[4] = -1;
  memset(sums, 0, 4 * sizeof(double));
  if (n < 3 || !(max_corr > 0.0) || ns < n || nt == 0) return;   /* rule 2 */
  int* s2t = (int*)malloc(sizeof(int) * (size_t)ns);
  int* t2s = (int*)malloc(sizeof(int) * (size_t)nt);
  or_feature_corr(sf, ns, tf, nt, s2t, t2s);
  int* cs = (int*)malloc(sizeof(int) * (size_t)ns);
  int* ct = (int*)malloc(sizeof(int) * (size_t)ns);
  int m = 0;
  if (mutual_filter) for (int i = 0; i < ns; i++) if (t2s[s2t[i]] == i) { cs[m] = i; ct[m] = s2t[i]; m++; }
  const int used_mutual = mutual_filter && m >= 3 * n;
  if (!used_mutual) { m = ns; for (int i = 0; i < ns; i++) { cs[i] = i; ct[i] = s2t[i]; } }
  stats[2] = m; stats[3] = used_mutual;
  void* tree = orc_kdtree_build(tx, nt);
  int64_t est_k = max_iteration, h = 0, validations = 0, best_h = -1;
  int best_inl = 0; double best_sum = 0.0, best_T[16], last_kd = 0.0;
  memcpy(best_T, T_out, sizeof(best_T));
  for (h = 0; h < est_k; h++) {
    double S[MAX_N][3], Q[MAX_N][3], T[16];
    for (int j = 0; j < n; j++) {
      const uint64_t k = or_stream(seed, h, n, j, (uint64_t)m);
      memcpy(S[j], sx + 3 * (size_t)cs[k], 24); memcpy(Q[j], tx + 3 * (size_t)ct[k], 24);
    }
    int ok = 1;   /* rule 5, edge length first */
    for (int i = 0; i < n && ok; i++) for (int j = i + 1; j < n && ok; j++) {
      const double ds = norm3(S[i][0] - S[j][0], S[i][1] - S[j][1], S[i][2] - S[j][2]);
      const double dt = norm3(Q[i][0] - Q[j][0], Q[i][1] - Q[j][1], Q[i][2] - Q[j][2]);
      if (ds < dt * checker_edge || dt < ds * checker_edge) ok = 0;
    }
    if (!ok) continue;
    umeyama((const double(*)[3])S, (const double(*)[3])Q, n, T);
    for (int j = 0; j < n && ok; j++) {
      double p[3];
      xform(T, S[j], p);
      if (norm3(Q[j][0] - p[0], Q[j][1] - p[1], Q[j][2] - p[2]) > checker_dist) ok = 0;
    }
    if (!ok) continue;
    /* rule 6 */
    validations++;
    int inl = 0; double sum = 0.0;
    for (int i = 0; i < ns; i++) {
      double q[3], d2; int idx;
      xform(T, sx + 3 * (size_t)i, q);
      if (orc_kdtree_search_hybrid(tree, q, max_corr, 1, &d2, &idx) > 0) { inl++; sum += d2; }
    }
    /* rule 7 */
    if (inl > 0 && (inl > best_inl || (inl == best_inl && sum < best_sum))) {
      best_inl = inl; best_sum = sum; best_h = h; memcpy(best_T, T, sizeof(T));
      const double fitness = (double)inl / (double)ns;
      const double k_d = log(1.0 - confidence) / log(1.0 - pow(fitness, (double)n));
      last_kd = k_d;
      if (k_d < (double)est_k) est_k = (int64_t)ceil(k_d);
    }
  }
  stats[0] = h; stats[1] = validations; stats[4] = best_h; stats[5] = best_inl;
  memcpy(T_out, best_T, sizeof(best_T));
  sums[0] = best_sum;
  sums[1] = best_inl > 0 ? (double)best_inl / (double)ns : 0.0;
  sums[2] = best_inl > 0 ? sqrt(best_sum / (double)best_inl) : 0.0;
  sums[3] = last_kd;
  orc_kdtree_free(tree);
  free(s2t); free(t2s); free(cs); free(ct);
}
