/* CPU restatement of the score of b2s_submap_global_localization (include/b2s.h, step 3) for the tests: hits(h) for every hypothesis
 * of the grid, OpenMP over the hypotheses.  Occupancy is a byte per voxel over the key range of the live map points; the numpy twin in
 * oracle_global_localization.py uses a set of packed keys instead.  Compiled with -ffp-contract=off: every product and sum is rounded
 * on its own, in the order the header states. */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define KEY_LIMIT 1048575.0   /* |floor(p / voxel)| must stay below 2^20 - 1 on every axis */

static int key_of(double x, double y, double z, double inv, long long k[3]) {
  const double f[3] = {floor(x * inv), floor(y * inv), floor(z * inv)};
  for (int d = 0; d < 3; d++) {
    if (!(fabs(f[d]) < KEY_LIMIT)) return 0;
    k[d] = (long long)f[d];
  }
  return 1;
}

/* map: nm x 3 live points; rot: n_yaw x 9 row-major; hits: nx ny n_yaw n_z.  Returns 0, or -1 when the occupancy does not fit. */
int gl_scores(const double* q, int nq, const double* map, int nm, const double* rot, double x_min, double y_min, double step, double z0,
              double z_step, int nx, int ny, int n_yaw, int n_z, double voxel, int32_t* hits) {
  const double inv = 1.0 / voxel;
  long long lo[3] = {0, 0, 0}, hi[3] = {-1, -1, -1};
  int any = 0;
  for (int i = 0; i < nm; i++) {
    long long k[3];
    if (!key_of(map[3 * i], map[3 * i + 1], map[3 * i + 2], inv, k)) continue;
    for (int d = 0; d < 3; d++) {
      if (!any || k[d] < lo[d]) lo[d] = k[d];
      if (!any || k[d] > hi[d]) hi[d] = k[d];
    }
    any = 1;
  }
  long long dim[3] = {0, 0, 0};
  size_t cells = 1;
  for (int d = 0; d < 3; d++) { dim[d] = any ? hi[d] - lo[d] + 1 : 0; cells *= (size_t)dim[d]; }
  if (cells > ((size_t)1 << 34)) return -1;
  unsigned char* occ = calloc(cells ? cells : 1, 1);
  if (!occ) return -1;
  for (int i = 0; i < nm; i++) {
    long long k[3];
    if (!key_of(map[3 * i], map[3 * i + 1], map[3 * i + 2], inv, k)) continue;
    occ[((size_t)(k[2] - lo[2]) * dim[1] + (size_t)(k[1] - lo[1])) * dim[0] + (size_t)(k[0] - lo[0])] = 1;
  }
  double* rq = malloc(sizeof(double) * 3 * (size_t)(nq > 0 ? nq : 1) * (size_t)n_yaw);
  for (int j = 0; j < n_yaw; j++) {
    const double* R = rot + 9 * j;
    for (int i = 0; i < nq; i++) {
      const double x = q[3 * i], y = q[3 * i + 1], z = q[3 * i + 2];
      double* o = rq + 3 * ((size_t)j * nq + i);
      o[0] = (R[0] * x + R[1] * y) + R[2] * z;
      o[1] = (R[3] * x + R[4] * y) + R[5] * z;
      o[2] = (R[6] * x + R[7] * y) + R[8] * z;
    }
  }
  const long long total = (long long)nx * ny * n_yaw * n_z;
#pragma omp parallel for schedule(dynamic, 4096)
  for (long long h = 0; h < total; h++) {
    const int ix = (int)(h % nx);
    long long r = h / nx;
    const int iy = (int)(r % ny);
    r /= ny;
    const int j = (int)(r % n_yaw), iz = (int)(r / n_yaw);
    const double tx = x_min + (double)ix * step, ty = y_min + (double)iy * step, tz = z0 + (double)iz * z_step;
    const double* o = rq + 3 * (size_t)j * nq;
    int c = 0;
    for (int i = 0; i < nq; i++) {
      long long k[3];
      if (!key_of(o[3 * i] + tx, o[3 * i + 1] + ty, o[3 * i + 2] + tz, inv, k)) continue;
      if (k[0] < lo[0] || k[0] > hi[0] || k[1] < lo[1] || k[1] > hi[1] || k[2] < lo[2] || k[2] > hi[2]) continue;
      c += occ[((size_t)(k[2] - lo[2]) * dim[1] + (size_t)(k[1] - lo[1])) * dim[0] + (size_t)(k[0] - lo[0])];
    }
    hits[h] = c;
  }
  free(rq);
  free(occ);
  return 0;
}
