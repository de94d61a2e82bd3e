/*
 * oracle_features.c -- CPU restatement of [O3D] v0.15.1 ComputeFPFHFeature (pipelines/registration/Feature.cpp), the feature
 * step of Submap::computeFeatures (core/src/Submap.cpp:244).  TEST INFRASTRUCTURE ONLY, like oracle/o3d_oracle.c, whose
 * KD-tree supplies the neighbour lists (orc_kdtree_search_hybrid: the k nearest with d2 < r2, ascending (d2, index)).
 * Restated from the published algorithm (Open3D's source is not available here); the assumptions are listed in DESIGN.md,
 * row K-fpfh.  Compiled with -ffp-contract=off: every expression is evaluated as written.
 */
#include <math.h>
#include <stdlib.h>
#include <string.h>

void* orc_kdtree_build(const double* pts, int n);
void orc_kdtree_free(void* t);
int orc_kdtree_search_hybrid(void* t, const double* q, double radius, int max_nn, double* d2, int* idx);

#define FO_PI 3.14159265358979323846

/* ComputePairFeatures: f[0] = atan2 angle, f[1] = v . n2, f[2] = angle1 (or -angle2 after the swap); zero for coincident points
 * and for a zero cross product.  *swap_margin = |acos|angle1| - acos|angle2||, how close the swap decision was. */
static void pair_features(const double* p1, const double* n1, const double* p2, const double* n2, double f[3], double* swap_margin) {
  double dp[3] = {p2[0] - p1[0], p2[1] - p1[1], p2[2] - p1[2]};
  const double len = sqrt(dp[0] * dp[0] + dp[1] * dp[1] + dp[2] * dp[2]);
  f[0] = f[1] = f[2] = 0.0;
  *swap_margin = INFINITY;
  if (len == 0.0) return;
  const double* a = n1; const double* b = n2;
  const double angle1 = (n1[0] * dp[0] + n1[1] * dp[1] + n1[2] * dp[2]) / len;
  const double angle2 = (n2[0] * dp[0] + n2[1] * dp[1] + n2[2] * dp[2]) / len;
  const double c1 = acos(fabs(angle1)), c2 = acos(fabs(angle2));
  *swap_margin = fabs(c1 - c2);
  double f2;
  if (c1 > c2) {
    a = n2; b = n1;
    dp[0] *= -1.0; dp[1] *= -1.0; dp[2] *= -1.0;
    f2 = -angle2;
  } else {
    f2 = angle1;
  }
  double v[3] = {dp[1] * a[2] - dp[2] * a[1], dp[2] * a[0] - dp[0] * a[2], dp[0] * a[1] - dp[1] * a[0]};
  const double vn = sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
  if (vn == 0.0) return;
  v[0] /= vn; v[1] /= vn; v[2] /= vn;
  const double w[3] = {a[1] * v[2] - a[2] * v[1], a[2] * v[0] - a[0] * v[2], a[0] * v[1] - a[1] * v[0]};
  f[2] = f2;
  f[1] = v[0] * b[0] + v[1] * b[1] + v[2] * b[2];
  f[0] = atan2(w[0] * b[0] + w[1] * b[1] + w[2] * b[2], a[0] * b[0] + a[1] * b[1] + a[2] * b[2]);
}

/* bin = floor(t) clamped to [0, 10]; *margin = distance of t to the nearest boundary that changes the bin (1 .. 10) */
static int bin_of(double t, double* margin) {
  double m = INFINITY;
  for (int k = 1; k <= 10; k++) { double e = fabs(t - (double)k); if (e < m) m = e; }
  if (m < *margin) *margin = m;
  int h = (int)floor(t);
  if (h < 0) h = 0;
  if (h >= 11) h = 10;
  return h;
}

/* feature: n x 33 (point after point).  Optional outputs: spfh (n x 33); margin (n): the smallest bin-boundary or swap margin over
 * the pairs of the point's SPFH; nb_idx / nb_d2 (n x knn) and nb_cnt (n): the hybrid neighbour lists. */
int fo_fpfh(const double* xyz, const double* nrm, int n, double radius, int knn, double* feature, double* spfh_out, double* margin,
            int* nb_idx_out, double* nb_d2_out, int* nb_cnt_out) {
  if (n <= 0) return 0;
  if (knn <= 0 || !(radius > 0.0)) return -1;
  int* nb_idx = (int*)malloc(sizeof(int) * (size_t)n * (size_t)knn);
  double* nb_d2 = (double*)malloc(sizeof(double) * (size_t)n * (size_t)knn);
  int* nb_cnt = (int*)malloc(sizeof(int) * (size_t)n);
  double* spfh = (double*)calloc((size_t)n * 33, sizeof(double));
  void* tree = orc_kdtree_build(xyz, n);
  for (int i = 0; i < n; i++)
    nb_cnt[i] = orc_kdtree_search_hybrid(tree, xyz + 3 * (size_t)i, radius, knn, nb_d2 + (size_t)i * knn, nb_idx + (size_t)i * knn);
  orc_kdtree_free(tree);
  /* ComputeSPFHFeature: only points with neighbours; element 0 of the list is skipped as the point itself */
  for (int i = 0; i < n; i++) {
    double mg = INFINITY;
    const int cnt = nb_cnt[i];
    if (cnt > 1) {
      const double hist_incr = 100.0 / (double)(cnt - 1);
      double* row = spfh + (size_t)i * 33;
      for (int k = 1; k < cnt; k++) {
        const int j = nb_idx[(size_t)i * knn + k];
        double f[3], sm;
        pair_features(xyz + 3 * (size_t)i, nrm + 3 * (size_t)i, xyz + 3 * (size_t)j, nrm + 3 * (size_t)j, f, &sm);
        if (sm < mg) mg = sm;
        row[bin_of(11 * (f[0] + FO_PI) / (2.0 * FO_PI), &mg)] += hist_incr;
        row[11 + bin_of(11 * (f[1] + 1.0) * 0.5, &mg)] += hist_incr;
        row[22 + bin_of(11 * (f[2] + 1.0) * 0.5, &mg)] += hist_incr;
      }
    }
    if (margin) margin[i] = mg;
  }
  /* ComputeFPFHFeature: spfh[nb] / d2 in neighbour order (d2 == 0 skipped), every 11-bin block scaled to 100, own SPFH added */
  for (int i = 0; i < n; i++) {
    double* out = feature + (size_t)i * 33;
    memset(out, 0, 33 * sizeof(double));
    const int cnt = nb_cnt[i];
    if (cnt <= 1) continue;
    double sum[3] = {0.0, 0.0, 0.0};
    for (int k = 1; k < cnt; k++) {
      const double dist = nb_d2[(size_t)i * knn + k];
      if (dist == 0.0) continue;
      const double* s = spfh + (size_t)nb_idx[(size_t)i * knn + k] * 33;
      for (int j = 0; j < 33; j++) {
        const double val = s[j] / dist;
        sum[j / 11] += val;
        out[j] += val;
      }
    }
    for (int j = 0; j < 3; j++) if (sum[j] != 0.0) sum[j] = 100.0 / sum[j];
    for (int j = 0; j < 33; j++) {
      out[j] *= sum[j / 11];
      out[j] += spfh[(size_t)i * 33 + j];
    }
  }
  if (spfh_out) memcpy(spfh_out, spfh, sizeof(double) * (size_t)n * 33);
  if (nb_idx_out) memcpy(nb_idx_out, nb_idx, sizeof(int) * (size_t)n * (size_t)knn);
  if (nb_d2_out) memcpy(nb_d2_out, nb_d2, sizeof(double) * (size_t)n * (size_t)knn);
  if (nb_cnt_out) memcpy(nb_cnt_out, nb_cnt, sizeof(int) * (size_t)n);
  free(nb_idx); free(nb_d2); free(nb_cnt); free(spfh);
  return 0;
}
