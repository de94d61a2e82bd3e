/*
 * oracle_submap_features.c -- CPU restatement of the feature-cloud front end of Submap::computeFeatures
 * (core/src/Submap.cpp:239-244): VoxelDownSample with the normals averaged, [O3D] v0.15.1 EstimateNormals on a cloud that
 * already has normals, NormalizeNormals, OrientNormalsTowardsCameraLocation(0), then ComputeFPFHFeature (fo_fpfh of
 * tests/oracle_features.c, linked into the same test library).  TEST INFRASTRUCTURE ONLY, like oracle/o3d_oracle.c, whose
 * KD-tree (orc_kdtree_search_hybrid), voxel down-sample and eigen-solver (orc_fast_eigen3x3) it uses; orc_estimate_normals, the
 * no-normals restatement, stays as it is.  Restated from the published algorithm (Open3D's source is not available here); the
 * assumptions are listed in DESIGN.md, row K-features.  Compiled with -ffp-contract=off: every expression is evaluated as written.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

void* orc_kdtree_build(const double* pts, int n);
void orc_kdtree_free(void* t);
int orc_kdtree_search_hybrid(void* t, const double* q, double radius, int max_nn, double* d2, int* idx);
size_t orc_voxel_down_sample(const double* xyz, const double* nrm, size_t n, double voxel, double* out_xyz, double* out_nrm, int32_t* out_keys);
void orc_fast_eigen3x3(const double cov[9], double* out);
int fo_fpfh(const double* xyz, const double* nrm, int n, double radius, int knn, double* feature, double* spfh_out, double* margin,
            int* nb_idx_out, double* nb_d2_out, int* nb_cnt_out);

/* [O3D] EstimateNormals(KDTreeSearchParamHybrid(radius, knn)) + NormalizeNormals + OrientNormalsTowardsCameraLocation(0), with the
 * branch orc_estimate_normals leaves out: prior (optional, n x 3) is the cloud's normals on entry.  With a prior a zero solver
 * result keeps the prior (instead of (0,0,1)), any other result is flipped when it points against the prior.  tie (optional, n):
 * 1 where the camera orientation was an exact tie, n . (-p) == 0, the only case in which the prior's sign survives. */
void fo_estimate_normals(const double* xyz, int n, int knn, double radius, const double* prior, double* out, int* tie) {
  if (n <= 0) return;
  void* tree = orc_kdtree_build(xyz, n);
  double* d2 = (double*)malloc(sizeof(double) * (size_t)knn);
  int* idx = (int*)malloc(sizeof(int) * (size_t)knn);
  for (int i = 0; i < n; i++) {
    const double* q = xyz + 3 * (size_t)i;
    double cov[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};   /* fewer than 3 neighbours: identity */
    const int k = orc_kdtree_search_hybrid(tree, q, radius, knn, d2, idx);
    if (k >= 3) {   /* utility::ComputeCovariance: single-pass cumulants in the search order */
      double c[9] = {0};
      for (int j = 0; j < k; j++) {
        const double* p = xyz + 3 * (size_t)idx[j];
        c[0] += p[0]; c[1] += p[1]; c[2] += p[2];
        c[3] += p[0] * p[0]; c[4] += p[0] * p[1]; c[5] += p[0] * p[2];
        c[6] += p[1] * p[1]; c[7] += p[1] * p[2]; c[8] += p[2] * p[2];
      }
      for (int j = 0; j < 9; j++) c[j] /= (double)k;
      cov[0] = c[3] - c[0] * c[0]; cov[4] = c[6] - c[1] * c[1]; cov[8] = c[8] - c[2] * c[2];
      cov[1] = cov[3] = c[4] - c[0] * c[1]; cov[2] = cov[6] = c[5] - c[0] * c[2]; cov[5] = cov[7] = c[7] - c[1] * c[2];
    }
    double nr[3];
    orc_fast_eigen3x3(cov, nr);
    const int zero = sqrt(nr[0] * nr[0] + nr[1] * nr[1] + nr[2] * nr[2]) == 0.0;
    if (prior) {
      const double* pv = prior + 3 * (size_t)i;
      if (zero) { nr[0] = pv[0]; nr[1] = pv[1]; nr[2] = pv[2]; }
      else if (nr[0] * pv[0] + nr[1] * pv[1] + nr[2] * pv[2] < 0.0) { nr[0] *= -1.0; nr[1] *= -1.0; nr[2] *= -1.0; }
    } else if (zero) { nr[0] = 0; nr[1] = 0; nr[2] = 1; }
    /* NormalizeNormals: a zero vector stays zero, NaN -> (0,0,1) */
    const double z = nr[0] * nr[0] + nr[1] * nr[1] + nr[2] * nr[2];
    if (z > 0) { const double s = sqrt(z); nr[0] /= s; nr[1] /= s; nr[2] /= s; }
    if (isnan(nr[0])) { nr[0] = 0; nr[1] = 0; nr[2] = 1; }
    /* OrientNormalsTowardsCameraLocation(camera = 0) */
    const double ref[3] = {-q[0], -q[1], -q[2]};
    int t = 0;
    if (sqrt(nr[0] * nr[0] + nr[1] * nr[1] + nr[2] * nr[2]) == 0.0) {
      const double rn = sqrt(ref[0] * ref[0] + ref[1] * ref[1] + ref[2] * ref[2]);
      if (rn == 0.0) { nr[0] = 0; nr[1] = 0; nr[2] = 1; }
      else { nr[0] = ref[0] / rn; nr[1] = ref[1] / rn; nr[2] = ref[2] / rn; }
    } else {
      const double dp = nr[0] * ref[0] + nr[1] * ref[1] + nr[2] * ref[2];
      if (dp < 0.0) { nr[0] *= -1.0; nr[1] *= -1.0; nr[2] *= -1.0; }
      t = dp == 0.0;
    }
    if (tie) tie[i] = t;
    memcpy(out + 3 * (size_t)i, nr, sizeof(nr));
  }
  free(d2); free(idx);
  orc_kdtree_free(tree);
}

/* Submap::computeFeatures, feature half (Submap.cpp:239-244): sparse = VoxelDownSample(map, voxel) with the normals averaged
 * (nrm may be NULL: a cloud without normals, estimated without priors and sp_prior left untouched), its normals with the
 * voxel-mean normals as priors, then ComputeFPFHFeature.
 * Outputs hold n points (the sparse cloud is never larger than the map): sparse xyz / prior normals / normals / voxel keys /
 * tie flags / features, plus the fo_fpfh details.  Returns the sparse size. */
int fo_submap_features(const double* xyz, const double* nrm, int n, double voxel, double normal_radius, int normal_knn, double feature_radius,
                       int feature_knn, double* sp_xyz, double* sp_prior, double* sp_nrm, int32_t* sp_keys, int* tie, double* feature,
                       double* spfh, double* margin, int* nb_idx, double* nb_d2, int* nb_cnt) {
  if (n <= 0) return 0;
  const int m = (int)orc_voxel_down_sample(xyz, nrm, (size_t)n, voxel, sp_xyz, nrm ? sp_prior : NULL, sp_keys);
  fo_estimate_normals(sp_xyz, m, normal_knn, normal_radius, nrm ? sp_prior : NULL, sp_nrm, tie);
  if (fo_fpfh(sp_xyz, sp_nrm, m, feature_radius, feature_knn, feature, spfh, margin, nb_idx, nb_d2, nb_cnt) != 0) return -1;
  return m;
}
